"""Numpy restatement of the GPU H.264 encoder (include/lspv.h): Constrained Baseline, I_16x16 and P_L0_16x16 / P_Skip
macroblocks, full-pel motion, CAVLC, no deblocking filter.  Written from ITU-T H.264 (clauses 7, 8.3, 8.4, 8.5, 9.2
and Annex A) and the encoder decisions fixed in lspv.h.

Every stage is exposed, so the GPU encoder (livespeechportraits_b200/h264.py) can be pinned stage by stage:
``to_yuv`` -> ``intra_mb`` / ``motion_search`` + ``inter_mb`` -> ``frame_bits`` (CAVLC) -> ``access_unit`` (NAL
packing).  ``encode`` runs a clip and returns the access units and the reconstructed planes, which a conforming decoder
reproduces exactly; ``max_bytes`` is the bound behind ``lspv_max_bytes``.

Inputs are uint8 ``[H, W, 3]`` RGB or ``[H, W]`` grey with H and W multiples of 16.
"""
from __future__ import annotations

import dataclasses
import math
from typing import List, Optional, Tuple

import numpy as np

# ---- tables --------------------------------------------------------------------------------------------------------

# lambda[QP] of the motion cost, round(sqrt(0.85 * 2^((QP - 12) / 3)))
LAMBDA = [0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 4, 4, 5, 5, 6, 7, 7, 8, 9, 10, 12,
          13, 15, 17, 19, 21, 23, 26, 30, 33, 37, 42, 47, 53, 59, 66, 74, 83]
MF = np.array([[13107, 5243, 8066], [11916, 4660, 7490], [10082, 4194, 6554], [9362, 3647, 5825], [8192, 3355, 5243],
               [7282, 2893, 4559]], np.int64)                               # forward quantisation multipliers
V = np.array([[10, 16, 13], [11, 18, 14], [13, 20, 16], [14, 23, 18], [16, 25, 20], [18, 29, 23]], np.int64)  # 8-315
CLS = np.array([[0, 2, 0, 2], [2, 1, 2, 1], [0, 2, 0, 2], [2, 1, 2, 1]])    # position class of (row, col)
ZIGZAG = np.array([0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15])  # scan index -> raster index (x + 4 y)
CHROMA_QP = list(range(30)) + [29, 30, 31, 32, 32, 33, 34, 34, 35, 35, 36, 36, 37, 37, 37, 38, 38, 38, 39, 39, 39, 39]
LEVEL_MAX = 2063              # the largest |level| CAVLC codes with level_prefix <= 15 under every suffixLength
BLK_XY = [(0, 0), (1, 0), (0, 1), (1, 1), (2, 0), (3, 0), (2, 1), (3, 1),
          (0, 2), (1, 2), (0, 3), (1, 3), (2, 2), (3, 2), (2, 3), (3, 3)]   # luma4x4BlkIdx -> (x, y) in 4x4 blocks
CF = np.array([[1, 1, 1, 1], [2, 1, -1, -2], [1, -1, -1, 1], [1, -2, 2, -1]], np.int64)
HAD4 = np.array([[1, 1, 1, 1], [1, 1, -1, -1], [1, -1, -1, 1], [1, -1, 1, -1]], np.int64)
HAD2 = np.array([[1, 1], [1, -1]], np.int64)

# Table 9-5, indexed [nC class][4 * TotalCoeff + TrailingOnes]: (length, code)
_CT_LEN = [
    [1, 0, 0, 0, 6, 2, 0, 0, 8, 6, 3, 0, 9, 8, 7, 5, 10, 9, 8, 6, 11, 10, 9, 7, 13, 11, 10, 8, 13, 13, 11, 9, 13, 13, 13,
     10, 14, 14, 13, 11, 14, 14, 14, 13, 15, 15, 14, 14, 15, 15, 15, 14, 16, 15, 15, 15, 16, 16, 16, 15, 16, 16, 16, 16,
     16, 16, 16, 16],
    [2, 0, 0, 0, 6, 2, 0, 0, 6, 5, 3, 0, 7, 6, 6, 4, 8, 6, 6, 4, 8, 7, 7, 5, 9, 8, 8, 6, 11, 9, 9, 6, 11, 11, 11, 7, 12,
     11, 11, 9, 12, 12, 12, 11, 12, 12, 12, 11, 13, 13, 13, 12, 13, 13, 13, 13, 13, 14, 13, 13, 14, 14, 14, 13, 14, 14,
     14, 14],
    [4, 0, 0, 0, 6, 4, 0, 0, 6, 5, 4, 0, 6, 5, 5, 4, 7, 5, 5, 4, 7, 5, 5, 4, 7, 6, 6, 4, 7, 6, 6, 4, 8, 7, 7, 5, 8, 8, 7,
     6, 9, 8, 8, 7, 9, 9, 8, 8, 9, 9, 9, 8, 10, 9, 9, 9, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10],
    [6, 0, 0, 0] + [6, 6, 0, 0] + [6, 6, 6, 0] + [6] * 56,
]
_CT_CODE = [
    [1, 0, 0, 0, 5, 1, 0, 0, 7, 4, 1, 0, 7, 6, 5, 3, 7, 6, 5, 3, 7, 6, 5, 4, 15, 6, 5, 4, 11, 14, 5, 4, 8, 10, 13, 4, 15,
     14, 9, 4, 11, 10, 13, 12, 15, 14, 9, 12, 11, 10, 13, 8, 15, 1, 9, 12, 11, 14, 13, 8, 7, 10, 9, 12, 4, 6, 5, 8],
    [3, 0, 0, 0, 11, 2, 0, 0, 7, 7, 3, 0, 7, 10, 9, 5, 7, 6, 5, 4, 4, 6, 5, 6, 7, 6, 5, 8, 15, 6, 5, 4, 11, 14, 13, 4,
     15, 10, 9, 4, 11, 14, 13, 12, 8, 10, 9, 8, 15, 14, 13, 12, 11, 10, 9, 12, 7, 11, 6, 8, 9, 8, 10, 1, 7, 6, 5, 4],
    [15, 0, 0, 0, 15, 14, 0, 0, 11, 15, 13, 0, 8, 12, 14, 12, 15, 10, 11, 11, 11, 8, 9, 10, 9, 14, 13, 9, 8, 10, 9, 8,
     15, 14, 13, 13, 11, 14, 10, 12, 15, 10, 13, 12, 11, 14, 9, 12, 8, 10, 13, 8, 13, 7, 9, 12, 9, 12, 11, 10, 5, 8, 7,
     6, 1, 4, 3, 2],
    [3, 0, 0, 0] + [0, 1, 0, 0] + [4, 5, 6, 0] + list(range(8, 64)),
]
_CDC_LEN = [2, 0, 0, 0, 6, 1, 0, 0, 6, 6, 3, 0, 6, 7, 7, 6, 6, 8, 8, 7]        # chroma DC (nC = -1)
_CDC_CODE = [1, 0, 0, 0, 7, 1, 0, 0, 4, 6, 1, 0, 3, 3, 2, 5, 2, 3, 2, 0]
# Tables 9-7 and 9-8, indexed [TotalCoeff - 1][total_zeros]
_TZ_LEN = [[1, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 9], [3, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 6, 6, 6, 6],
           [4, 3, 3, 3, 4, 4, 3, 3, 4, 5, 5, 6, 5, 6], [5, 3, 4, 4, 3, 3, 3, 4, 3, 4, 5, 5, 5],
           [4, 4, 4, 3, 3, 3, 3, 3, 4, 5, 4, 5], [6, 5, 3, 3, 3, 3, 3, 3, 4, 3, 6], [6, 5, 3, 3, 3, 2, 3, 4, 3, 6],
           [6, 4, 5, 3, 2, 2, 3, 3, 6], [6, 6, 4, 2, 2, 3, 2, 5], [5, 5, 3, 2, 2, 2, 4], [4, 4, 3, 3, 1, 3],
           [4, 4, 2, 1, 3], [3, 3, 1, 2], [2, 2, 1], [1, 1]]
_TZ_CODE = [[1, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 1], [7, 6, 5, 4, 3, 5, 4, 3, 2, 3, 2, 3, 2, 1, 0],
            [5, 7, 6, 5, 4, 3, 4, 3, 2, 3, 2, 1, 1, 0], [3, 7, 5, 4, 6, 5, 4, 3, 3, 2, 2, 1, 0],
            [5, 4, 3, 7, 6, 5, 4, 3, 2, 1, 1, 0], [1, 1, 7, 6, 5, 4, 3, 2, 1, 1, 0], [1, 1, 5, 4, 3, 3, 2, 1, 1, 0],
            [1, 1, 1, 3, 3, 2, 2, 1, 0], [1, 0, 1, 3, 2, 1, 1, 1], [1, 0, 1, 3, 2, 1, 1], [0, 1, 1, 2, 1, 3],
            [0, 1, 1, 1, 1], [0, 1, 1, 1], [0, 1, 1], [0, 1]]
_CTZ_LEN = [[1, 2, 3, 3], [1, 2, 2], [1, 1]]                                  # chroma DC, [TotalCoeff - 1][total_zeros]
_CTZ_CODE = [[1, 1, 1, 0], [1, 1, 0], [1, 0]]
# Table 9-10, indexed [min(zerosLeft, 7) - 1][run_before]
_RB_LEN = [[1, 1], [1, 2, 2], [2, 2, 2, 2], [2, 2, 2, 3, 3], [2, 2, 3, 3, 3, 3], [2, 3, 3, 3, 3, 3, 3],
           [3, 3, 3, 3, 3, 3, 3, 4, 5, 6, 7, 8, 9, 10, 11]]
_RB_CODE = [[1, 0], [1, 1, 0], [3, 2, 1, 0], [3, 2, 1, 1, 0], [3, 2, 3, 2, 1, 0], [3, 0, 1, 3, 2, 5, 4],
            [7, 6, 5, 4, 3, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1]]
# Table 9-4 (chroma_format_idc 1): codeNum -> coded_block_pattern of Inter macroblocks
INTER_CBP = [0, 16, 1, 2, 4, 8, 32, 3, 5, 10, 12, 15, 47, 7, 11, 13, 14, 6, 9, 31, 35, 37, 42, 44, 33, 34, 36, 40, 39,
             43, 45, 46, 17, 18, 20, 24, 19, 21, 26, 28, 23, 27, 29, 30, 22, 25, 38, 41]
INTER_CBP_CODE = [INTER_CBP.index(c) for c in range(48)]
# Table A-1: (level_idc, MaxMBPS, MaxFS, MaxDpbMbs)
LEVELS = [(10, 1485, 99, 396), (11, 3000, 396, 900), (12, 6000, 396, 2376), (13, 11880, 396, 2376),
          (20, 11880, 396, 2376), (21, 19800, 792, 4752), (22, 20250, 1620, 8100), (30, 40500, 1620, 8100),
          (31, 108000, 3600, 18000), (32, 216000, 5120, 20480), (40, 245760, 8192, 32768), (41, 245760, 8192, 32768),
          (42, 522240, 8704, 34816), (50, 589824, 22080, 110400), (51, 983040, 36864, 184320),
          (52, 2073600, 36864, 184320), (60, 4177920, 139264, 696320), (61, 8355840, 139264, 696320),
          (62, 16711680, 139264, 696320)]


# ---- colour ----------------------------------------------------------------------------------------------------------

def to_yuv(img: np.ndarray) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """BT.601 limited-range Y'CbCr 4:2:0 planes (uint8) of an RGB ``[H, W, 3]`` or grey ``[H, W]`` uint8 image."""
    if img.ndim == 2:
        img = np.repeat(img[:, :, None], 3, axis=2)
    r, g, b = (img[:, :, k].astype(np.int64) for k in range(3))
    y = ((66 * r + 129 * g + 25 * b + 128) >> 8) + 16
    cb = ((-38 * r - 74 * g + 112 * b + 128) >> 8) + 128
    cr = ((112 * r - 94 * g - 18 * b + 128) >> 8) + 128

    def sub(c):
        return (c[0::2, 0::2] + c[0::2, 1::2] + c[1::2, 0::2] + c[1::2, 1::2] + 2) >> 2
    return y.astype(np.uint8), sub(cb).astype(np.uint8), sub(cr).astype(np.uint8)


# ---- transforms, quantisation, scaling (8.5) -------------------------------------------------------------------------

def forward4(x: np.ndarray) -> np.ndarray:
    """The forward core transform Cf X Cf^T of a 4x4 residual."""
    return CF @ x.astype(np.int64) @ CF.T


def _quant(w, mf, shift, f):
    return np.clip(np.sign(w) * ((np.abs(w) * mf + f) >> shift), -LEVEL_MAX, LEVEL_MAX)


def quant4(w: np.ndarray, qp: int, intra: bool) -> np.ndarray:
    """Levels of a 4x4 coefficient block: sign(W) (|W| MF + f) >> qbits, f = 2^qbits / 3 intra, / 6 inter, clamped."""
    qbits = 15 + qp // 6
    return _quant(w, MF[qp % 6][CLS], qbits, (1 << qbits) // (3 if intra else 6))


def quant_dc(w: np.ndarray, qp: int, intra: bool) -> np.ndarray:
    """Levels of a DC block (luma 4x4 after the halved Hadamard, chroma 2x2): sign (|W| MF00 + 2 f) >> (qbits + 1)."""
    qbits = 15 + qp // 6
    return _quant(w, MF[qp % 6][0], qbits + 1, 2 * ((1 << qbits) // (3 if intra else 6)))


def dequant4(c: np.ndarray, qp: int) -> np.ndarray:
    """8.5.12.1 with flat scaling lists: c LevelScale4x4 scaled by 2^(qP/6 - 4), which is c v 2^(qP/6) exactly."""
    return (c * V[qp % 6][CLS]) << (qp // 6)


def inverse4(d: np.ndarray) -> np.ndarray:
    """8.5.12.2: rows, then columns, then (h + 32) >> 6."""
    def core(a0, a1, a2, a3):
        e0, e1, e2, e3 = a0 + a2, a0 - a2, (a1 >> 1) - a3, a1 + (a3 >> 1)
        return e0 + e3, e1 + e2, e1 - e2, e0 - e3
    d = d.astype(np.int64)
    f = np.stack(core(d[:, 0], d[:, 1], d[:, 2], d[:, 3]), axis=1)
    g = np.stack(core(f[0], f[1], f[2], f[3]), axis=0)
    return (g + 32) >> 6


def luma_dc_scale(c: np.ndarray, qp: int) -> np.ndarray:
    """8.5.10: the Intra16x16 DC levels (4x4, [block y][block x]) -> dcY."""
    f = HAD4 @ c @ HAD4
    ls = 16 * V[qp % 6][0]
    if qp >= 36:
        return (f * ls) << (qp // 6 - 6)
    return (f * ls + (1 << (5 - qp // 6))) >> (6 - qp // 6)


def chroma_dc_scale(c: np.ndarray, qpc: int) -> np.ndarray:
    """8.5.11.2 for 4:2:0: the 2x2 chroma DC levels -> dcC."""
    return ((HAD2 @ c @ HAD2) * (16 * V[qpc % 6][0]) << (qpc // 6)) >> 5


# ---- intra prediction (8.3.3, 8.3.4) ---------------------------------------------------------------------------------

def luma_preds(rec: np.ndarray, mx: int, my: int) -> dict:
    """The Intra_16x16 predictions the neighbours allow: mode (0 V, 1 H, 2 DC, 3 Plane) -> 16x16 int64."""
    x0, y0 = 16 * mx, 16 * my
    top = rec[y0 - 1, x0:x0 + 16].astype(np.int64) if my else None
    left = rec[y0:y0 + 16, x0 - 1].astype(np.int64) if mx else None
    out = {}
    if top is not None:
        out[0] = np.tile(top, (16, 1))
    if left is not None:
        out[1] = np.tile(left[:, None], (1, 16))
    if top is not None and left is not None:
        dc = (top.sum() + left.sum() + 16) >> 5
    elif left is not None:
        dc = (left.sum() + 8) >> 4
    elif top is not None:
        dc = (top.sum() + 8) >> 4
    else:
        dc = 128
    out[2] = np.full((16, 16), dc, np.int64)
    if top is not None and left is not None:
        tl = int(rec[y0 - 1, x0 - 1])
        t, l = np.concatenate([[tl], top]), np.concatenate([[tl], left])       # index k: p[k - 1, -1] / p[-1, k - 1]
        h = sum((i + 1) * (t[9 + i] - t[7 - i]) for i in range(8))
        v = sum((i + 1) * (l[9 + i] - l[7 - i]) for i in range(8))
        a, b, c = 16 * (left[15] + top[15]), (5 * h + 32) >> 6, (5 * v + 32) >> 6
        yy, xx = np.mgrid[0:16, 0:16]
        out[3] = np.clip((a + b * (xx - 7) + c * (yy - 7) + 16) >> 5, 0, 255)
    return out


def chroma_preds(rec: np.ndarray, mx: int, my: int) -> dict:
    """The intra chroma predictions of one 8x8 component: mode (0 DC, 1 H, 2 V, 3 Plane) -> 8x8 int64."""
    x0, y0 = 8 * mx, 8 * my
    top = rec[y0 - 1, x0:x0 + 8].astype(np.int64) if my else None
    left = rec[y0:y0 + 8, x0 - 1].astype(np.int64) if mx else None
    dc = np.zeros((8, 8), np.int64)
    for by in range(2):
        for bx in range(2):
            st = top[4 * bx:4 * bx + 4].sum() if top is not None else None
            sl = left[4 * by:4 * by + 4].sum() if left is not None else None
            if bx == by:                                  # (0, 0) and (4, 4): both, else either
                v = (st + sl + 4) >> 3 if st is not None and sl is not None else \
                    (sl + 2) >> 2 if sl is not None else (st + 2) >> 2 if st is not None else 128
            elif by == 0:                                 # (4, 0): top first
                v = (st + 2) >> 2 if st is not None else (sl + 2) >> 2 if sl is not None else 128
            else:                                         # (0, 4): left first
                v = (sl + 2) >> 2 if sl is not None else (st + 2) >> 2 if st is not None else 128
            dc[4 * by:4 * by + 4, 4 * bx:4 * bx + 4] = v
    out = {0: dc}
    if left is not None:
        out[1] = np.tile(left[:, None], (1, 8))
    if top is not None:
        out[2] = np.tile(top, (8, 1))
    if top is not None and left is not None:
        tl = int(rec[y0 - 1, x0 - 1])
        t, l = np.concatenate([[tl], top]), np.concatenate([[tl], left])
        h = sum((i + 1) * (t[5 + i] - t[3 - i]) for i in range(4))
        v = sum((i + 1) * (l[5 + i] - l[3 - i]) for i in range(4))
        a, b, c = 16 * (left[7] + top[7]), (34 * h + 32) >> 6, (34 * v + 32) >> 6
        yy, xx = np.mgrid[0:8, 0:8]
        out[3] = np.clip((a + b * (xx - 3) + c * (yy - 3) + 16) >> 5, 0, 255)
    return out


# ---- macroblocks -----------------------------------------------------------------------------------------------------

@dataclasses.dataclass
class Mb:
    """One macroblock's decisions and levels.  ``luma[b]`` holds block b's (luma4x4BlkIdx) levels in scan order: 16 for
    P (all coded), 16 with index 0 unused for I_16x16 (whose DC levels are ``dc``).  ``cdc[c]`` / ``cac[c][b]`` are the
    chroma DC levels (raster order of the 2x2) and the AC levels (scan positions 1..15 at 1..15) of Cb (c 0) and Cr."""
    intra: bool
    mode: int = 0                  # Intra_16x16 prediction mode
    cmode: int = 0                 # intra_chroma_pred_mode
    mv: Tuple[int, int] = (0, 0)   # full-pel (x, y)
    dc: Optional[np.ndarray] = None
    luma: Optional[np.ndarray] = None
    cdc: Optional[np.ndarray] = None
    cac: Optional[np.ndarray] = None
    skip: bool = False

    @property
    def cbp_luma(self) -> int:
        if self.intra:
            return 15 if np.any(self.luma[:, 1:]) else 0
        return sum(1 << i for i in range(4) if np.any(self.luma[4 * i:4 * i + 4]))

    @property
    def cbp_chroma(self) -> int:
        return 2 if np.any(self.cac[:, :, 1:]) else 1 if np.any(self.cdc) else 0


def _code_luma(res: np.ndarray, qp: int, intra: bool):
    """Residual 16x16 -> (dc levels scan order or None, [16 blocks][16] levels scan order, reconstructed residual)."""
    w = np.zeros((4, 4, 4, 4), np.int64)                        # [by][bx] of 4x4 coefficient blocks
    for by in range(4):
        for bx in range(4):
            w[by, bx] = forward4(res[4 * by:4 * by + 4, 4 * bx:4 * bx + 4])
    lev = np.zeros((4, 4, 4, 4), np.int64)
    for by in range(4):
        for bx in range(4):
            lev[by, bx] = quant4(w[by, bx], qp, intra)
    dc = None
    if intra:
        dcl = quant_dc((HAD4 @ w[:, :, 0, 0] @ HAD4) >> 1, qp, True)
        dc = dcl.reshape(16)[ZIGZAG]
        dcy = luma_dc_scale(dcl, qp)
        lev[:, :, 0, 0] = 0
    out = np.zeros((16, 16), np.int64)
    scan = np.zeros((16, 16), np.int64)
    for b, (bx, by) in enumerate(BLK_XY):
        scan[b] = lev[by, bx].reshape(16)[ZIGZAG]
        d = dequant4(lev[by, bx], qp)
        if intra:
            d[0, 0] = dcy[by, bx]
        out[4 * by:4 * by + 4, 4 * bx:4 * bx + 4] = inverse4(d)
    return dc, scan, out


def _code_chroma(res: np.ndarray, qpc: int, intra: bool):
    """Residual 8x8 of one component -> (dc levels [4], ac levels [4][16] scan order, reconstructed residual)."""
    w = np.zeros((2, 2, 4, 4), np.int64)
    for by in range(2):
        for bx in range(2):
            w[by, bx] = forward4(res[4 * by:4 * by + 4, 4 * bx:4 * bx + 4])
    dcl = quant_dc(HAD2 @ w[:, :, 0, 0] @ HAD2, qpc, intra)
    dcc = chroma_dc_scale(dcl, qpc)
    ac = np.zeros((4, 16), np.int64)
    out = np.zeros((8, 8), np.int64)
    for by in range(2):
        for bx in range(2):
            lev = quant4(w[by, bx], qpc, intra)
            lev[0, 0] = 0
            ac[2 * by + bx] = lev.reshape(16)[ZIGZAG]
            d = dequant4(lev, qpc)
            d[0, 0] = dcc[by, bx]
            out[4 * by:4 * by + 4, 4 * bx:4 * bx + 4] = inverse4(d)
    return dcl.reshape(4), ac, out


def _sad(a, b) -> int:
    return int(np.abs(a.astype(np.int64) - b).sum())


def intra_mb(src, rec, mx: int, my: int, qp: int) -> Mb:
    """Codes macroblock (mx, my) as I_16x16 against the reconstructed neighbours in ``rec`` (three planes, updated in
    place).  The mode of least SAD wins, the lowest mode number on ties; chroma SAD is Cb's plus Cr's."""
    y0, x0 = 16 * my, 16 * mx
    s = src[0][y0:y0 + 16, x0:x0 + 16]
    preds = luma_preds(rec[0], mx, my)
    mode = min(preds, key=lambda m: (_sad(s, preds[m]), m))
    dc, luma, r = _code_luma(s.astype(np.int64) - preds[mode], qp, True)
    rec[0][y0:y0 + 16, x0:x0 + 16] = np.clip(preds[mode] + r, 0, 255)
    qpc = CHROMA_QP[qp]
    cs = [src[k][8 * my:8 * my + 8, 8 * mx:8 * mx + 8] for k in (1, 2)]
    cp = [chroma_preds(rec[k], mx, my) for k in (1, 2)]
    cmode = min(cp[0], key=lambda m: (_sad(cs[0], cp[0][m]) + _sad(cs[1], cp[1][m]), m))
    cdc, cac = np.zeros((2, 4), np.int64), np.zeros((2, 4, 16), np.int64)
    for k in range(2):
        cdc[k], cac[k], r = _code_chroma(cs[k].astype(np.int64) - cp[k][cmode], qpc, True)
        rec[k + 1][8 * my:8 * my + 8, 8 * mx:8 * mx + 8] = np.clip(cp[k][cmode] + r, 0, 255)
    return Mb(True, mode, cmode, (0, 0), dc, luma, cdc, cac)


def se_bits(v: int) -> int:
    """Length of the se(v) code of v."""
    k = 2 * v - 1 if v > 0 else -2 * v
    return 2 * (k + 1).bit_length() - 1


def motion_search(cur: np.ndarray, ref: np.ndarray, qp: int, search: int) -> np.ndarray:
    """Full-pel vectors [mbh, mbw, 2] (x, y): per macroblock the least SAD + lambda[QP] (se bits of 4 dx and 4 dy), over
    |dx|, |dy| <= search with the 16x16 block inside the frame; ties go to the smaller dy, then the smaller dx."""
    h, w = cur.shape
    mbh, mbw = h // 16, w // 16
    pad = np.zeros((h + 2 * search, w + 2 * search), np.int64)
    pad[search:search + h, search:search + w] = ref
    c = cur.astype(np.int64)
    best = np.full((mbh, mbw), np.iinfo(np.int64).max, np.int64)
    mv = np.zeros((mbh, mbw, 2), np.int64)
    ys, xs = np.arange(mbh)[:, None] * 16, np.arange(mbw)[None, :] * 16
    for dy in range(-search, search + 1):
        for dx in range(-search, search + 1):
            sh = pad[search + dy:search + dy + h, search + dx:search + dx + w]
            sad = np.abs(c - sh).reshape(mbh, 16, mbw, 16).sum(axis=(1, 3))
            cost = sad + LAMBDA[qp] * (se_bits(4 * dx) + se_bits(4 * dy))
            ok = (ys + dy >= 0) & (ys + dy + 16 <= h) & (xs + dx >= 0) & (xs + dx + 16 <= w)
            better = ok & (cost < best)
            best = np.where(better, cost, best)
            mv[better] = (dx, dy)
    return mv


def chroma_mc(ref: np.ndarray, mx: int, my: int, dx: int, dy: int) -> np.ndarray:
    """8.4.2.2.2: the 8x8 chroma prediction of macroblock (mx, my) for full-pel luma vector (dx, dy) (chroma vector 4 dx,
    4 dy in eighth samples), with edge clamping."""
    hc, wc = ref.shape
    fx, fy = (4 * dx) & 7, (4 * dy) & 7
    yy, xx = np.mgrid[0:8, 0:8]
    xi, yi = 8 * mx + ((4 * dx) >> 3) + xx, 8 * my + ((4 * dy) >> 3) + yy
    r = ref.astype(np.int64)

    def at(y, x):
        return r[np.clip(y, 0, hc - 1), np.clip(x, 0, wc - 1)]
    return ((8 - fx) * (8 - fy) * at(yi, xi) + fx * (8 - fy) * at(yi, xi + 1) + (8 - fx) * fy * at(yi + 1, xi) +
            fx * fy * at(yi + 1, xi + 1) + 32) >> 6


def inter_mb(src, ref, rec, mx: int, my: int, mv, qp: int) -> Mb:
    """Codes macroblock (mx, my) as P_L0_16x16 with vector ``mv`` from the previous reconstruction ``ref``; the
    reconstruction goes to ``rec``.  Whether it becomes P_Skip is decided by ``frame_bits`` from the neighbours."""
    dx, dy = int(mv[0]), int(mv[1])
    y0, x0 = 16 * my, 16 * mx
    pred = ref[0][y0 + dy:y0 + dy + 16, x0 + dx:x0 + dx + 16].astype(np.int64)
    _, luma, r = _code_luma(src[0][y0:y0 + 16, x0:x0 + 16].astype(np.int64) - pred, qp, False)
    rec[0][y0:y0 + 16, x0:x0 + 16] = np.clip(pred + r, 0, 255)
    qpc = CHROMA_QP[qp]
    cdc, cac = np.zeros((2, 4), np.int64), np.zeros((2, 4, 16), np.int64)
    for k in range(2):
        p = chroma_mc(ref[k + 1], mx, my, dx, dy)
        cdc[k], cac[k], r = _code_chroma(src[k + 1][8 * my:8 * my + 8, 8 * mx:8 * mx + 8].astype(np.int64) - p, qpc,
                                         False)
        rec[k + 1][8 * my:8 * my + 8, 8 * mx:8 * mx + 8] = np.clip(p + r, 0, 255)
    return Mb(False, mv=(dx, dy), luma=luma, cdc=cdc, cac=cac)


# ---- bit writing and CAVLC (9.2) -------------------------------------------------------------------------------------

class BitWriter:
    def __init__(self):
        self.parts: List[str] = []
        self.n = 0

    def u(self, n: int, v: int) -> None:
        if n:
            self.parts.append(format(v, f"0{n}b"))
            self.n += n

    def ue(self, v: int) -> None:
        k = (v + 1).bit_length()
        self.u(k - 1, 0)
        self.u(k, v + 1)

    def se(self, v: int) -> None:
        self.ue(2 * v - 1 if v > 0 else -2 * v)

    def bits(self) -> str:
        return "".join(self.parts)


def rbsp_bytes(bits: str) -> bytes:
    """rbsp_trailing_bits: a 1, then zeros to the byte boundary."""
    bits += "1" + "0" * (-(len(bits) + 1) % 8)
    return int(bits, 2).to_bytes(len(bits) // 8, "big")


def emulation_prevention(rbsp: bytes) -> bytes:
    """00 00 0x (x <= 3) -> 00 00 03 0x."""
    out, zeros = bytearray(), 0
    for b in rbsp:
        if zeros >= 2 and b <= 3:
            out.append(3)
            zeros = 0
        out.append(b)
        zeros = zeros + 1 if b == 0 else 0
    return bytes(out)


def nal(header: int, rbsp: bytes) -> bytes:
    return b"\x00\x00\x00\x01" + bytes([header]) + emulation_prevention(rbsp)


def coeff_token_class(nc: int) -> int:
    return 0 if nc < 2 else 1 if nc < 4 else 2 if nc < 8 else 3


def residual_block(w: BitWriter, coef, nc: int) -> int:
    """residual_block_cavlc of the levels ``coef`` (scan order, maxNumCoeff = len(coef)) with context nC (-1: chroma
    DC).  Returns TotalCoeff."""
    coef = [int(c) for c in coef]
    nz = [i for i, c in enumerate(coef) if c]
    tc = len(nz)
    t1 = 0
    for i in reversed(nz):
        if abs(coef[i]) != 1 or t1 == 3:
            break
        t1 += 1
    if nc == -1:
        w.u(_CDC_LEN[4 * tc + t1], _CDC_CODE[4 * tc + t1])
    else:
        k = coeff_token_class(nc)
        w.u(_CT_LEN[k][4 * tc + t1], _CT_CODE[k][4 * tc + t1])
    if tc == 0:
        return 0
    levels = [coef[i] for i in reversed(nz)]
    for k in range(t1):
        w.u(1, 1 if levels[k] < 0 else 0)
    sl = 1 if tc > 10 and t1 < 3 else 0
    for k in range(t1, tc):
        lv = levels[k]
        code = 2 * lv - 2 if lv > 0 else -2 * lv - 1
        if k == t1 and t1 < 3:
            code -= 2
        if sl == 0:
            if code < 14:
                prefix, suffix, size = code, 0, 0
            elif code < 30:
                prefix, suffix, size = 14, code - 14, 4
            else:
                prefix, suffix, size = 15, code - 30, 12
        elif code < (15 << sl):
            prefix, suffix, size = code >> sl, code & ((1 << sl) - 1), sl
        else:
            prefix, suffix, size = 15, code - (15 << sl), 12
        assert suffix < (1 << size) or size == suffix == 0, (lv, sl)
        w.u(prefix + 1, 1)
        w.u(size, suffix)
        if sl == 0:
            sl = 1
        if abs(lv) > (3 << (sl - 1)) and sl < 6:
            sl += 1
    tz = nz[-1] + 1 - tc
    if tc < len(coef):
        if len(coef) == 4:
            w.u(_CTZ_LEN[tc - 1][tz], _CTZ_CODE[tc - 1][tz])
        else:
            w.u(_TZ_LEN[tc - 1][tz], _TZ_CODE[tc - 1][tz])
    left = tz
    for k in range(tc - 1, 0, -1):
        if left <= 0:
            break
        run = nz[k] - nz[k - 1] - 1
        t = min(left, 7) - 1
        w.u(_RB_LEN[t][run], _RB_CODE[t][run])
        left -= run
    return tc


def _nc(grid: np.ndarray, y: int, x: int) -> int:
    a = grid[y, x - 1] if x > 0 else None
    b = grid[y - 1, x] if y > 0 else None
    if a is not None and b is not None:
        return (int(a) + int(b) + 1) >> 1
    return int(a) if a is not None else int(b) if b is not None else 0


def median(a, b, c):
    return max(min(a, b), min(max(a, b), c))


def mv_pred(mvs: np.ndarray, mx: int, my: int) -> Tuple[Tuple[int, int], Tuple[int, int]]:
    """(mvp of 8.4.1.3, P_Skip vector of 8.4.1.1) of 16x16 macroblock (mx, my) in quarter samples, from the final
    vectors ``mvs`` [mbh, mbw, 2] (quarter samples) of a P slice without intra macroblocks."""
    mbh, mbw = mvs.shape[:2]

    def nb(x, y):
        return (True, tuple(int(v) for v in mvs[y, x])) if 0 <= x < mbw and 0 <= y < mbh else (False, (0, 0))
    a, b = nb(mx - 1, my), nb(mx, my - 1)
    c = nb(mx + 1, my - 1)
    if not c[0]:
        c = nb(mx - 1, my - 1)
    if not b[0] and not c[0] and a[0]:
        b = c = a
    avail = [n for n in (a, b, c) if n[0]]
    if len(avail) == 1:
        mvp = avail[0][1]
    else:
        mvp = (median(a[1][0], b[1][0], c[1][0]), median(a[1][1], b[1][1], c[1][1]))
    na, nbb = nb(mx - 1, my), nb(mx, my - 1)
    if not na[0] or not nbb[0] or na[1] == (0, 0) or nbb[1] == (0, 0):
        skip = (0, 0)
    else:
        skip = mvp
    return mvp, skip


def frame_bits(mbs: List[List[Mb]], idr: bool, w: BitWriter) -> None:
    """slice_data() of one frame of decided macroblocks (P_Skip is decided here) into ``w``."""
    mbh, mbw = len(mbs), len(mbs[0])
    tcl = np.zeros((4 * mbh, 4 * mbw), np.int64)
    tcc = np.zeros((2, 2 * mbh, 2 * mbw), np.int64)
    for my in range(mbh):
        for mx in range(mbw):
            m = mbs[my][mx]
            for b, (bx, by) in enumerate(BLK_XY):
                tcl[4 * my + by, 4 * mx + bx] = np.count_nonzero(m.luma[b][1:] if m.intra else m.luma[b])
            for k in range(2):
                for b in range(4):
                    tcc[k, 2 * my + b // 2, 2 * mx + b % 2] = np.count_nonzero(m.cac[k, b, 1:])
    mvs = np.array([[[4 * m.mv[0], 4 * m.mv[1]] for m in row] for row in mbs], np.int64)
    run = 0
    for my in range(mbh):
        for mx in range(mbw):
            m = mbs[my][mx]
            cbpl, cbpc = m.cbp_luma, m.cbp_chroma
            if not idr:
                mvp, skip = mv_pred(mvs, mx, my)
                if tuple(mvs[my, mx]) == skip and cbpl == 0 and cbpc == 0:
                    m.skip = True
                    run += 1
                    continue
                w.ue(run)
                run = 0
                w.ue(0)                                                           # P_L0_16x16
                w.se(int(mvs[my, mx, 0]) - mvp[0])
                w.se(int(mvs[my, mx, 1]) - mvp[1])
                w.ue(INTER_CBP_CODE[cbpl | cbpc << 4])
                if cbpl == 0 and cbpc == 0:
                    continue
                w.se(0)                                                           # mb_qp_delta
                for b, (bx, by) in enumerate(BLK_XY):
                    if cbpl >> (b // 4) & 1:
                        residual_block(w, m.luma[b], _nc(tcl, 4 * my + by, 4 * mx + bx))
            else:
                w.ue(1 + m.mode + 4 * cbpc + (12 if cbpl else 0))
                w.ue(m.cmode)
                w.se(0)
                residual_block(w, m.dc, _nc(tcl, 4 * my, 4 * mx))
                if cbpl:
                    for b, (bx, by) in enumerate(BLK_XY):
                        residual_block(w, m.luma[b][1:], _nc(tcl, 4 * my + by, 4 * mx + bx))
            if cbpc:
                for k in range(2):
                    residual_block(w, m.cdc[k], -1)
            if cbpc == 2:
                for k in range(2):
                    for b in range(4):
                        residual_block(w, m.cac[k, b, 1:], _nc(tcc[k], 2 * my + b // 2, 2 * mx + b % 2))
    if run:
        w.ue(run)


# ---- parameter sets, slice header, access unit (7.3) -----------------------------------------------------------------

def level_idc(height: int, width: int, fps: int) -> int:
    """The lowest level of Table A-1 whose MaxFS, MaxMBPS, MaxDpbMbs (one reference frame) and frame dimension limit
    sqrt(8 MaxFS) fit; 0 if none does.  Bit rate is not constrained."""
    fs, mbw, mbh = (height // 16) * (width // 16), width // 16, height // 16
    for idc, mbps, maxfs, dpb in LEVELS:
        if fs <= maxfs and mbw * mbw <= 8 * maxfs and mbh * mbh <= 8 * maxfs and fs * fps <= mbps and fs <= dpb:
            return idc
    return 0


def sps(height: int, width: int, fps: int) -> bytes:
    w = BitWriter()
    w.u(8, 66)
    w.u(8, 0xC0)                                 # constraint_set0_flag, constraint_set1_flag: Constrained Baseline
    w.u(8, level_idc(height, width, fps))
    w.ue(0)                                      # seq_parameter_set_id
    w.ue(0)                                      # log2_max_frame_num_minus4
    w.ue(2)                                      # pic_order_cnt_type
    w.ue(1)                                      # max_num_ref_frames
    w.u(1, 0)                                    # gaps_in_frame_num_value_allowed_flag
    w.ue(width // 16 - 1)
    w.ue(height // 16 - 1)
    w.u(1, 1)                                    # frame_mbs_only_flag
    w.u(1, 1)                                    # direct_8x8_inference_flag
    w.u(1, 0)                                    # frame_cropping_flag
    w.u(1, 1)                                    # vui_parameters_present_flag
    w.u(1, 0)                                    # aspect_ratio_info_present_flag
    w.u(1, 0)                                    # overscan_info_present_flag
    w.u(1, 1)                                    # video_signal_type_present_flag
    w.u(3, 5)                                    # video_format: unspecified
    w.u(1, 0)                                    # video_full_range_flag: limited
    w.u(1, 1)                                    # colour_description_present_flag
    w.u(8, 6)                                    # colour_primaries: SMPTE 170M
    w.u(8, 6)                                    # transfer_characteristics: SMPTE 170M
    w.u(8, 6)                                    # matrix_coefficients: SMPTE 170M (BT.601)
    w.u(1, 0)                                    # chroma_loc_info_present_flag
    w.u(1, 1)                                    # timing_info_present_flag
    w.u(32, 1)                                   # num_units_in_tick
    w.u(32, 2 * fps)                             # time_scale
    w.u(1, 1)                                    # fixed_frame_rate_flag
    w.u(1, 0)                                    # nal_hrd_parameters_present_flag
    w.u(1, 0)                                    # vcl_hrd_parameters_present_flag
    w.u(1, 0)                                    # pic_struct_present_flag
    w.u(1, 1)                                    # bitstream_restriction_flag
    w.u(1, 1)                                    # motion_vectors_over_pic_boundaries_flag
    w.ue(0)                                      # max_bytes_per_pic_denom
    w.ue(0)                                      # max_bits_per_mb_denom
    w.ue(16)                                     # log2_max_mv_length_horizontal
    w.ue(16)                                     # log2_max_mv_length_vertical
    w.ue(0)                                      # max_num_reorder_frames
    w.ue(1)                                      # max_dec_frame_buffering
    return rbsp_bytes(w.bits())


def pps() -> bytes:
    w = BitWriter()
    w.ue(0)                                      # pic_parameter_set_id
    w.ue(0)                                      # seq_parameter_set_id
    w.u(1, 0)                                    # entropy_coding_mode_flag: CAVLC
    w.u(1, 0)                                    # bottom_field_pic_order_in_frame_present_flag
    w.ue(0)                                      # num_slice_groups_minus1
    w.ue(0)                                      # num_ref_idx_l0_default_active_minus1
    w.ue(0)                                      # num_ref_idx_l1_default_active_minus1
    w.u(1, 0)                                    # weighted_pred_flag
    w.u(2, 0)                                    # weighted_bipred_idc
    w.se(0)                                      # pic_init_qp_minus26
    w.se(0)                                      # pic_init_qs_minus26
    w.se(0)                                      # chroma_qp_index_offset
    w.u(1, 1)                                    # deblocking_filter_control_present_flag
    w.u(1, 0)                                    # constrained_intra_pred_flag
    w.u(1, 0)                                    # redundant_pic_cnt_present_flag
    return rbsp_bytes(w.bits())


def slice_header(w: BitWriter, frame: int, gop: int, qp: int) -> None:
    idr = frame % gop == 0
    w.ue(0)                                      # first_mb_in_slice
    w.ue(7 if idr else 5)                        # slice_type: I / P, every slice of the picture alike
    w.ue(0)                                      # pic_parameter_set_id
    w.u(4, (frame % gop) % 16)                   # frame_num
    if idr:
        w.ue((frame // gop) & 1)                 # idr_pic_id, different for consecutive IDR pictures
    else:
        w.u(1, 0)                                # num_ref_idx_active_override_flag
        w.u(1, 0)                                # ref_pic_list_modification_flag_l0
    if idr:
        w.u(1, 0)                                # no_output_of_prior_pics_flag
        w.u(1, 0)                                # long_term_reference_flag
    else:
        w.u(1, 0)                                # adaptive_ref_pic_marking_mode_flag
    w.se(qp - 26)                                # slice_qp_delta
    w.ue(1)                                      # disable_deblocking_filter_idc


def access_unit(mbs, frame: int, gop: int, qp: int, height: int, width: int, fps: int) -> bytes:
    """SPS + PPS before an IDR slice, or one P slice; 4-byte start codes."""
    idr = frame % gop == 0
    w = BitWriter()
    slice_header(w, frame, gop, qp)
    frame_bits(mbs, idr, w)
    out = nal(0x67, sps(height, width, fps)) + nal(0x68, pps()) if idr else b""
    return out + nal(0x65 if idr else 0x61, rbsp_bytes(w.bits()))


# ---- the encoder -----------------------------------------------------------------------------------------------------

@dataclasses.dataclass
class State:
    """The encoder's carry between calls: the next frame index and the last reconstructed frame (Y, Cb, Cr)."""
    frame: int = 0
    ref: Optional[Tuple[np.ndarray, np.ndarray, np.ndarray]] = None


def encode_frame(img: np.ndarray, state: State, qp: int, gop: int, search: int, fps: int):
    """One access unit; advances ``state``.  Returns (bytes, is_idr, reconstruction (Y, Cb, Cr))."""
    h, w = img.shape[:2]
    src = to_yuv(img)
    rec = [np.zeros_like(p) for p in src]
    idr = state.frame % gop == 0
    mbh, mbw = h // 16, w // 16
    if idr:
        mbs = [[intra_mb(src, rec, mx, my, qp) for mx in range(mbw)] for my in range(mbh)]
    else:
        mv = motion_search(src[0], state.ref[0], qp, search)
        mbs = [[inter_mb(src, state.ref, rec, mx, my, mv[my, mx], qp) for mx in range(mbw)] for my in range(mbh)]
    au = access_unit(mbs, state.frame, gop, qp, h, w, fps)
    state.frame += 1
    state.ref = tuple(rec)
    return au, idr, state.ref


def encode(frames, qp: int = 26, gop: int = 60, search: int = 16, fps: int = 60, state: Optional[State] = None):
    """Encodes ``frames`` (a sequence of uint8 images) from ``state`` (None: a fresh stream).  Returns (access units,
    IDR flags, reconstructions, state)."""
    state = State() if state is None else state
    aus, idrs, recs = [], [], []
    for img in frames:
        au, idr, rec = encode_frame(np.asarray(img), state, qp, gop, search, fps)
        aus.append(au)
        idrs.append(idr)
        recs.append(rec)
    return aus, idrs, recs, state


# ---- the bound (include/lspv.h) --------------------------------------------------------------------------------------

def worst_block_bits(max_coeff: int) -> int:
    """coeff_token (16, chroma DC 8) + max_coeff levels of at most 28 bits (prefix 16 + suffix 12; a trailing-one sign is
    shorter) + total_zeros (9, chroma DC 3) + max_coeff - 1 run_before codes (11, chroma DC 2)."""
    if max_coeff == 4:
        return 8 + 4 * 28 + 3 + 3 * 2
    return 16 + max_coeff * 28 + 9 + (max_coeff - 1) * 11


def worst_mb_bits(mbs: int, search: int = 64) -> int:
    """Per macroblock: the larger of an I_16x16 and a P_L0_16x16 one, plus a mb_skip_run code of at most ue(mbs)."""
    chroma = 2 * worst_block_bits(4) + 8 * worst_block_bits(15)
    intra = 9 + 5 + 1 + worst_block_bits(16) + 16 * worst_block_bits(15) + chroma
    mvd = se_bits(-8 * search)                  # |mvd| <= 2 * 4 * search quarter samples
    inter = 1 + 2 * mvd + 11 + 1 + 16 * worst_block_bits(16) + chroma
    return max(intra, inter) + 2 * (mbs + 1).bit_length() - 1


def max_bytes(height: int, width: int) -> int:
    """lspv_max_bytes: SPS and PPS (at most 64 bytes each with their start codes), the slice NAL's start code and header
    byte, and the slice RBSP (a 64-bit slice header, the macroblocks, a trailing byte) with one emulation-prevention
    byte per two payload bytes at most."""
    mbs = (height // 16) * (width // 16)
    rbsp = (64 + mbs * worst_mb_bits(mbs) + 8 + 7) // 8
    return 2 * 64 + 5 + rbsp + (rbsp + 1) // 2
