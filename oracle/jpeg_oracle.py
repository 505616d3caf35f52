"""Numpy restatement of the baseline JPEG encoder PIL drives (``Image.save(f, "JPEG", quality=q)``): libjpeg-turbo's
jcparam (quality scaling with force_baseline, the standard Huffman tables), jccolor (rgb_ycc_convert's fixed-point
tables), jcsample (h2v2_downsample), jfdctint (islow), jcdctmgr (the rounding divide), jchuff (standard-table coding)
and jcmarker (the marker segments), written from the published algorithms.

Every stage is exposed, so the GPU encoder (livespeechportraits_b200/jpeg.py) can be pinned stage by stage:
``rgb_to_ycc`` -> ``downsample_h2v2`` -> ``fdct_islow`` -> ``quantize`` (zigzag order) -> ``block_bits`` -> ``encode``.
``worst_block_bits`` is the per-block worst case behind ``lspj_max_bytes`` (include/lspj.h).

Inputs are uint8 ``[H, W, 3]`` RGB or ``[H, W]`` grey with H and W multiples of 16, the sizes the encoder accepts.
"""
from __future__ import annotations

import numpy as np

# ---- jcparam: the standard tables (JPEG standard Annex K) ---------------------------------------------------------

LUMA_QUANT = np.array([
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
    14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], np.int64)     # natural order
CHROMA_QUANT = np.array([
    17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
    47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32, np.int64)

# zigzag position k -> natural (row-major) index: jpeg_natural_order
ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
    54, 47, 55, 62, 63], np.int64)

_AC_LUMA_VALS = bytes.fromhex(
    "01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25262728292a343536373839"
    "3a434445464748494a535455565758595a636465666768696a737475767778797a838485868788898a92939495969798999aa2a3a4a5a6a7"
    "a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7e8e9eaf1f2f3f4f5f6f7f8f9fa")
_AC_CHROMA_VALS = bytes.fromhex(
    "000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a162434e125f11718191a262728292a35363738"
    "393a434445464748494a535455565758595a636465666768696a737475767778797a82838485868788898a92939495969798999aa2a3a4a5"
    "a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5e6e7e8e9eaf2f3f4f5f6f7f8f9fa")

# (BITS[1..16], HUFFVAL) of the four standard tables, in jcmarker's DHT order: DC 0, AC 0, DC 1, AC 1
DC_LUMA = ((0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0), bytes(range(12)))
AC_LUMA = ((0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D), _AC_LUMA_VALS)
DC_CHROMA = ((0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0), bytes(range(12)))
AC_CHROMA = ((0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77), _AC_CHROMA_VALS)


def huffman_codes(table):
    """jchuff jpeg_make_c_derived_tbl: ``(code[256], size[256])`` of a (BITS, HUFFVAL) table; size 0 = no code."""
    bits, vals = table
    code = np.zeros(256, np.int64)
    size = np.zeros(256, np.int64)
    c, k = 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            code[vals[k]], size[vals[k]] = c, length
            c += 1
            k += 1
        c <<= 1
    return code, size


def quality_scaling(quality: int) -> int:
    """jpeg_quality_scaling."""
    quality = min(max(int(quality), 1), 100)
    return 5000 // quality if quality < 50 else 200 - quality * 2


def quant_tables(quality: int, components: int = 3):
    """jpeg_set_quality(quality, force_baseline=TRUE): the natural-order tables of the components' slots (luma, chroma)."""
    scale = quality_scaling(quality)
    out = []
    for basic in (LUMA_QUANT, CHROMA_QUANT)[:1 if components == 1 else 2]:
        out.append(np.clip((basic * scale + 50) // 100, 1, 255))
    return out


# ---- jccolor / jcsample ------------------------------------------------------------------------------------------

def _fix(x: float) -> int:
    return int(x * (1 << 16) + 0.5)


def rgb_to_ycc(img: np.ndarray):
    """rgb_ycc_convert: uint8 [H, W, 3] -> (Y, Cb, Cr) uint8 planes, SCALEBITS 16 fixed point."""
    r, g, b = (img[..., i].astype(np.int64) for i in range(3))
    half, cbcr = 1 << 15, 128 << 16
    y = (_fix(0.29900) * r + _fix(0.58700) * g + _fix(0.11400) * b + half) >> 16
    cb = (-_fix(0.16874) * r - _fix(0.33126) * g + _fix(0.5) * b + cbcr + half - 1) >> 16
    cr = (_fix(0.5) * r - _fix(0.41869) * g - _fix(0.08131) * b + cbcr + half - 1) >> 16
    return y.astype(np.uint8), cb.astype(np.uint8), cr.astype(np.uint8)


def downsample_h2v2(plane: np.ndarray) -> np.ndarray:
    """h2v2_downsample: 2x2 means with the bias alternating 1, 2, 1, 2, ... along each output row."""
    p = plane.astype(np.int64)
    s = p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2]
    bias = np.where(np.arange(s.shape[1]) % 2 == 0, 1, 2)
    return ((s + bias) >> 2).astype(np.uint8)


# ---- jfdctint / jcdctmgr -----------------------------------------------------------------------------------------

_C = {k: v for k, v in dict(c0298=2446, c0390=3196, c0541=4433, c0765=6270, c0899=7373, c1175=9633, c1501=12299,
                            c1847=15137, c1961=16069, c2053=16819, c2562=20995, c3072=25172).items()}


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_1d(d, pass1: bool):
    """One jfdctint pass over the last axis of d (int64 [..., 8])."""
    cb, pb = 13, 2
    t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    out = np.empty_like(d)
    sh = cb - pb if pass1 else cb + pb
    if pass1:
        out[..., 0], out[..., 4] = (t10 + t11) << pb, (t10 - t11) << pb
    else:
        out[..., 0], out[..., 4] = _descale(t10 + t11, pb), _descale(t10 - t11, pb)
    z1 = (t12 + t13) * _C["c0541"]
    out[..., 2] = _descale(z1 + t13 * _C["c0765"], sh)
    out[..., 6] = _descale(z1 - t12 * _C["c1847"], sh)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * _C["c1175"]
    t4, t5, t6, t7 = t4 * _C["c0298"], t5 * _C["c2053"], t6 * _C["c3072"], t7 * _C["c1501"]
    z1, z2 = z1 * -_C["c0899"], z2 * -_C["c2562"]
    z3, z4 = z3 * -_C["c1961"] + z5, z4 * -_C["c0390"] + z5
    out[..., 7] = _descale(t4 + z1 + z3, sh)
    out[..., 5] = _descale(t5 + z2 + z4, sh)
    out[..., 3] = _descale(t6 + z2 + z3, sh)
    out[..., 1] = _descale(t7 + z1 + z4, sh)
    return out


def fdct_islow(blocks: np.ndarray) -> np.ndarray:
    """jpeg_fdct_islow of uint8 sample blocks [N, 8, 8] (centred by 128 first, as convsamp does): int64 [N, 8, 8] in
    natural order, scaled up by 8 as islow leaves them."""
    d = blocks.astype(np.int64) - 128
    d = _fdct_1d(d, True)                                             # rows
    return np.swapaxes(_fdct_1d(np.swapaxes(d, 1, 2), False), 1, 2)   # columns


def quantize(coefs: np.ndarray, qtable: np.ndarray) -> np.ndarray:
    """jcdctmgr quantize: each coefficient divided by 8 * qtable, rounded half away from zero; int64 [N, 64] in
    zigzag order."""
    d = (qtable.astype(np.int64) * 8)[ZIGZAG]
    x = coefs.reshape(-1, 64)[:, ZIGZAG]
    q = (np.abs(x) + d // 2) // d
    return np.where(x < 0, -q, q)


def quantize_reciprocal(x: np.ndarray, divisor: int) -> np.ndarray:
    """libjpeg-turbo's quantize with 16-bit DCTELEM (its SIMD build): compute_reciprocal's (recip, corr, scale, shift),
    then ((|x| + corr) * recip >> 16) * scale >> 16, sign restored.  Pinned equal to ``quantize``'s divide by the tests."""
    b = int(divisor).bit_length() - 1
    r = 16 + b
    fq, fr = divmod(1 << r, divisor)
    c = divisor // 2
    if fr == 0:
        fq >>= 1
        r -= 1
    elif fr <= divisor // 2:
        c += 1
    else:
        fq += 1
    scale = 1 << (32 - r)
    a = np.abs(x.astype(np.int64))
    q = ((((a + c) & 0xFFFF) * fq >> 16) * scale) >> 16
    return np.where(x < 0, -q, q)


# ---- block order and Huffman coding -------------------------------------------------------------------------------

def scan_blocks(img: np.ndarray, quality: int):
    """The quantised zigzag blocks in scan order, int64 [nblocks, 64], with each block's component (0 Y, 1 Cb, 2 Cr).
    RGB: per 16x16 MCU in raster order, Y0 Y1 Y2 Y3 Cb Cr; grey: the 8x8 blocks in raster order."""
    img = np.asarray(img, np.uint8)
    h, w = img.shape[:2]
    if h % 16 or w % 16:
        raise ValueError("height and width must be multiples of 16")
    tabs = quant_tables(quality, 1 if img.ndim == 2 else 3)

    def blocks(plane):                                                 # [bh, bw, 8, 8]
        bh, bw = plane.shape[0] // 8, plane.shape[1] // 8
        return plane.reshape(bh, 8, bw, 8).swapaxes(1, 2)

    if img.ndim == 2:
        zz = quantize(fdct_islow(blocks(img).reshape(-1, 8, 8)), tabs[0])
        return zz, np.zeros(len(zz), np.int64)
    y, cb, cr = rgb_to_ycc(img)
    my, mx = h // 16, w // 16
    yb = blocks(y).reshape(my, 2, mx, 2, 8, 8).transpose(0, 2, 1, 3, 4, 5).reshape(my, mx, 4, 8, 8)
    cbb = blocks(downsample_h2v2(cb)).reshape(my, mx, 1, 8, 8)
    crb = blocks(downsample_h2v2(cr)).reshape(my, mx, 1, 8, 8)
    qy = quantize(fdct_islow(yb.reshape(-1, 8, 8)), tabs[0]).reshape(my, mx, 4, 64)
    qb = quantize(fdct_islow(cbb.reshape(-1, 8, 8)), tabs[1]).reshape(my, mx, 1, 64)
    qr = quantize(fdct_islow(crb.reshape(-1, 8, 8)), tabs[1]).reshape(my, mx, 1, 64)
    zz = np.concatenate([qy, qb, qr], axis=2).reshape(-1, 64)
    comp = np.tile(np.array([0, 0, 0, 0, 1, 2]), my * mx)
    return zz, comp


def dc_diffs(zz: np.ndarray, comp: np.ndarray) -> np.ndarray:
    """Per-component DC prediction in scan order, starting from 0."""
    diff = np.empty(len(zz), np.int64)
    for c in np.unique(comp):
        idx = np.nonzero(comp == c)[0]
        dc = zz[idx, 0]
        diff[idx] = dc - np.concatenate([[0], dc[:-1]])
    return diff


_TABLES = [tuple(tuple(a.tolist() for a in huffman_codes(t)) for t in pair)
           for pair in ((DC_LUMA, AC_LUMA), (DC_CHROMA, AC_CHROMA))]


def _symbols(row, dc_diff, table):
    """encode_one_block's (code, size) pairs for one block (a list of 64 zigzag ints), magnitudes included."""
    (dcc, dcs), (acc, acs) = _TABLES[table]
    n = abs(dc_diff).bit_length()
    out = [(dcc[n], dcs[n])]
    if n:
        out.append(((dc_diff - 1 if dc_diff < 0 else dc_diff) & ((1 << n) - 1), n))
    r = 0
    for k in range(1, 64):
        v = row[k]
        if v == 0:
            r += 1
            continue
        while r > 15:
            out.append((acc[0xF0], acs[0xF0]))
            r -= 16
        n = abs(v).bit_length()
        out.append((acc[(r << 4) + n], acs[(r << 4) + n]))
        out.append(((v - 1 if v < 0 else v) & ((1 << n) - 1), n))
        r = 0
    if r > 0:
        out.append((acc[0], acs[0]))
    return out


def _all_symbols(zz: np.ndarray, comp: np.ndarray):
    diff = dc_diffs(zz, comp).tolist()
    return [_symbols(row, d, int(c > 0)) for row, d, c in zip(zz.tolist(), diff, comp.tolist())]


def block_bits(zz: np.ndarray, comp: np.ndarray) -> np.ndarray:
    """Each block's Huffman-coded bit count (DC prediction included), int64 [nblocks]."""
    return np.array([sum(s for _, s in syms) for syms in _all_symbols(zz, comp)], np.int64)


def worst_block_bits() -> int:
    """The per-block bound behind lspj_max_bytes: the longest DC code plus 11 magnitude bits, 63 AC codes of at most
    16 + 10 bits, three ZRLs (63 // 16) of at most 16 bits and an EOB of at most 16 bits."""
    return 16 + 11 + 63 * (16 + 10) + 3 * 16 + 16


def scan_bytes(zz: np.ndarray, comp: np.ndarray) -> bytes:
    """The entropy-coded segment: bits MSB first, padded with 1 bits to a byte, every 0xFF followed by 0x00."""
    parts, nacc = [], 0
    for syms in _all_symbols(zz, comp):
        for code, size in syms:
            parts.append(format(code, "0%db" % size))
            nacc += size
    acc = int("".join(parts) or "0", 2)
    pad = (-nacc) % 8
    acc = (acc << pad) | ((1 << pad) - 1)
    raw = acc.to_bytes((nacc + pad) // 8, "big") if nacc + pad else b""
    return raw.replace(b"\xff", b"\xff\x00")


# ---- jcmarker -----------------------------------------------------------------------------------------------------

def _segment(marker: int, payload: bytes) -> bytes:
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + payload


def header(height: int, width: int, components: int, quality: int) -> bytes:
    """SOI, JFIF APP0 (1.01, no units, 1:1), DQT per table, SOF0, DHT per table (DC 0, AC 0, DC 1, AC 1) and SOS."""
    tabs = quant_tables(quality, components)
    out = b"\xff\xd8" + _segment(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for i, t in enumerate(tabs):
        out += _segment(0xDB, bytes([i]) + bytes(t[ZIGZAG].astype(np.uint8)))
    comps = [(1, 0x22, 0)] if components == 3 else [(1, 0x11, 0)]
    comps += [(2, 0x11, 1), (3, 0x11, 1)] if components == 3 else []
    sof = bytes([8]) + height.to_bytes(2, "big") + width.to_bytes(2, "big") + bytes([components])
    out += _segment(0xC0, sof + b"".join(bytes(c) for c in comps))
    for i, (dc, ac) in enumerate([(DC_LUMA, AC_LUMA), (DC_CHROMA, AC_CHROMA)][:len(tabs)]):
        out += _segment(0xC4, bytes([i]) + bytes(dc[0]) + dc[1])
        out += _segment(0xC4, bytes([0x10 | i]) + bytes(ac[0]) + ac[1])
    sos = bytes([components]) + b"".join(bytes([c, (t << 4) | t]) for c, _, t in comps) + b"\x00\x3f\x00"
    return out + _segment(0xDA, sos)


def encode(img: np.ndarray, quality: int = 75) -> bytes:
    """The complete .jpg file PIL writes for ``Image.fromarray(img).save(f, "JPEG", quality=quality)``."""
    img = np.asarray(img, np.uint8)
    zz, comp = scan_blocks(img, quality)
    return header(img.shape[0], img.shape[1], 1 if img.ndim == 2 else 3, quality) + scan_bytes(zz, comp) + b"\xff\xd9"


def max_bytes(height: int, width: int, components: int, quality: int = 100) -> int:
    """lspj_max_bytes restated: header + at most two bytes per scan byte (stuffing) of the worst-case scan + EOI."""
    nblocks = (height // 8) * (width // 8) * (1 if components == 1 else 6) // (1 if components == 1 else 4)
    scan = (nblocks * worst_block_bits() + 7) // 8
    return len(header(height, width, components, quality)) + 2 * scan + 2
