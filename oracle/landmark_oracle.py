"""Oracle of the landmark post-processing (row N7, demo.py stage 5, :215-255).

* ``stage5``: a restatement of demo.py:217-255 with funcs/utils.py's ``landmark_smooth_3d``, ``mouth_pts_AMP``,
  ``solve_intersect_mouth``, ``headpose_smooth``, ``angle2matrix`` and ``project_landmarks`` (scipy's
  ``gaussian_filter1d``, numpy).  It follows the numpy installed here: under numpy >= 2 ``scale * rot.dot(...)``
  with a float64 numpy scalar is float64, under numpy 1.18 (the reference's pin) it stayed fp32.  oracle/
  make_golden_landmarks.py asserts it bit-equal to the unmodified reference statements.
* ``truth``: float64 with no intermediate roundings, smoothing with its own reflect-rule filter ``gauss_reflect``.
* ``error_bound``: per-element bound on |kernel - truth| derived from the kernel's arithmetic (csrc/lspl.cu).
* ``emulate``: the kernel's steps in float64 with its fp32 roundings, with named defects (``MUTATIONS``) that the
  bound must catch.
* ``make_identity`` / ``make_tracks``: a seeded synthetic identity and tracks (nothing of data/ ships).
"""
from __future__ import annotations

import ast
import math
import os
import types
from typing import Optional

import numpy as np
from scipy.ndimage import gaussian_filter1d

from oracle.mel_oracle import REFERENCE_ROOT, UTILS_FILE

DEMO_FILE = os.path.join(REFERENCE_ROOT, "demo.py")
MOUTH_INDICES = np.concatenate([np.arange(4, 11), np.arange(46, 64)])                      # demo.py:74
EYE_BROW_INDICES = np.array([27, 65, 28, 68, 29, 67, 30, 66, 31, 72, 32, 69, 33, 70, 34, 71], np.int32)   # :75
UPPER_INNER, LOWER_INNER = [63, 62, 61], [58, 59, 60]                                     # funcs/utils.py:269-270
UPPER_OUTER, LOWER_OUTER = list(range(47, 52)), list(range(57, 52, -1))
UPPER_MOUTH = [46, 47, 48, 49, 50, 51, 52, 61, 62, 63]
LOWER_MOUTH = [53, 54, 55, 56, 57, 58, 59, 60]
U32 = 2.0 ** -24
U64 = 2.0 ** -53

# config/May.yaml and config/Obama1.yaml, under demo.py's names (:120-126)
MAY = dict(Feat_smooth_sigma=1.5, AMP_method="XYZ", Feat_AMPs=[2, 2, 2], rot_AMP=1, trans_AMP=0.5,
           Head_smooth_sigma=[5, 10], shoulder_AMP=0.5)
OBAMA1 = dict(Feat_smooth_sigma=1, AMP_method="XYZ", Feat_AMPs=[1.5, 1.5, 1.5], rot_AMP=1, trans_AMP=1,
              Head_smooth_sigma=[2, 8], shoulder_AMP=0.5)
IDENTITY_KEYS = ("mean_pts3d", "std_mean_pts3d", "candidate_eye_brow", "mean_translation", "ref_trans", "shoulder3D",
                 "camera_intrinsic", "scale")


# ------------------------------------------------------------------------------------------------------------------
# Synthetic identity and tracks
# ------------------------------------------------------------------------------------------------------------------
def make_identity(seed: int = 0, m: int = 37) -> dict:
    """A face of 73 points about 16 x 16 units, 60 units in front of a 1200-pixel camera centred in 512 x 512, so that
    every face point lands inside the image and the outer shoulder points outside it.  The mean face keeps the lower
    inner lip 0.6 below the upper one.  dtypes as demo.py loads them: fp32 files, ``scale`` a float64 numpy scalar."""
    rng = np.random.default_rng(seed)
    mean = np.zeros((73, 3))
    mean[:, 0] = rng.uniform(-7, 7, 73)
    mean[:, 1] = rng.uniform(-9, 7, 73)
    mean[:, 2] = rng.uniform(0, 4, 73)
    mean[46:64, 0] = np.linspace(-2.5, 2.5, 18)
    mean[46:64, 1] = -5.0 + rng.uniform(-0.1, 0.1, 18)
    mean[UPPER_OUTER, 1] = -4.2
    mean[LOWER_OUTER, 1] = -5.8
    mean[UPPER_INNER, 1] = -4.7
    mean[LOWER_INNER, 1] = -5.3
    mean = mean.astype(np.float32)
    pts3d = (mean + rng.normal(0, 0.15, (10 + m, 73, 3))).astype(np.float32)         # the identity's fitted landmarks
    trans = (np.float32([0.3, -0.8, 60.0]) + rng.normal(0, 0.4, (40, 3))).astype(np.float32)
    sh = np.zeros((18, 3), np.float32)
    for side, sgn in ((0, -1), (1, 1)):
        i = np.arange(9)
        sh[side * 9 + i, 0] = sgn * (5 + 1.9 * i)
        sh[side * 9 + i, 1] = 8 + 0.09 * i ** 2 + rng.uniform(0, 0.3, 9)
        sh[side * 9 + i, 2] = 62 + rng.uniform(-1, 1, 9)
    K = np.float32([[1200, 0, 255.5], [0, 1195, 256.25], [0, 0, 1]])
    return {"mean_pts3d": mean, "std_mean_pts3d": pts3d.mean(axis=0),
            "candidate_eye_brow": (pts3d - mean)[10:, EYE_BROW_INDICES], "mean_translation": trans.mean(axis=0),
            "ref_trans": trans[1], "shoulder3D": sh, "camera_intrinsic": K, "scale": np.float64(1.0375)}


def make_tracks(n_feat: int, n_head: int, seed: int = 0, cross: float = 0.1):
    """``pred_Feat`` [n_feat, 75] fp32 (mouth deltas) and ``pred_Head`` [n_head, 12] float64 holding fp32 values, as
    Audio2Feature / Audio2Headpose return them.  Inner-lip pair j crosses after an AMP a when
    ``open(t) g_j > 0.6 / a`` (g = 0.9, 1, 1.1): ``cross`` = 0.1 gives frames where all three pairs cross and frames
    where only some do at AMP 1.5 to 2; ``cross`` = -0.5 gives none."""
    rng = np.random.default_rng(seed)
    t = np.arange(n_feat, dtype=np.float64)
    feat = rng.normal(0, 0.05, (n_feat, 25, 3))
    feat[:, 7:] += 0.2 * np.sin(2 * np.pi * t[:, None, None] / 23 + rng.uniform(0, 6, (1, 18, 3)))
    openness = cross + 0.35 * np.sin(2 * np.pi * t / 37) + 0.15 * np.sin(2 * np.pi * t / 11.3 + 1) + rng.normal(0, 0.04, n_feat)
    g = np.array([0.9, 1.0, 1.1])
    for j in range(3):
        feat[:, 7 + UPPER_INNER[j] - 46, 1] -= openness * g[j] / 2
        feat[:, 7 + LOWER_INNER[j] - 46, 1] += openness * g[j] / 2
    for r in UPPER_OUTER:
        feat[:, 7 + r - 46, 1] -= 0.3 * openness
    for r in LOWER_OUTER:
        feat[:, 7 + r - 46, 1] += 0.3 * openness
    th = np.arange(n_head, dtype=np.float64)
    head = np.zeros((n_head, 12))
    for c in range(3):
        head[:, c] = 3 * np.sin(2 * np.pi * th / (97 + 13 * c) + c) + 2 * np.sin(2 * np.pi * th / 31) + rng.normal(0, 0.8, n_head)
    for c in range(3, 6):
        head[:, c] = 1.5 * np.sin(2 * np.pi * th / (150 + 20 * c)) + rng.normal(0, 0.3, n_head)
    head[:, 6:] = rng.normal(0, 1, (n_head, 6))
    return feat.reshape(n_feat, 75).astype(np.float32), head.astype(np.float32).astype(np.float64)


# ------------------------------------------------------------------------------------------------------------------
# Restatement of demo.py:217-255 (scipy / numpy, the reference's operations in its order)
# ------------------------------------------------------------------------------------------------------------------
def mouth_pts_AMP(pts3d, is_delta=True, method="XY", paras=(1, 1)):   # noqa: N802 - funcs/utils.py:274
    if method == "XY" and is_delta:
        pts3d[:, 46:64, 0] *= paras[0]
        pts3d[:, 46:64, 1] *= paras[1]
    elif method == "XYZ" and is_delta:
        for c in range(3):
            pts3d[:, 46:64, c] *= paras[c]
    elif method == "LowerMore" and is_delta:
        for c in range(3):
            pts3d[:, UPPER_MOUTH, c] *= paras[c]
        for c in range(3):
            pts3d[:, LOWER_MOUTH, c] *= paras[3 + c]
    else:
        raise NotImplementedError(method)
    return pts3d


def solve_intersect_mouth(pts3d):
    lower_inner_y, upper_inner_y = pts3d[:, LOWER_INNER, 1], pts3d[:, UPPER_INNER, 1]
    flip = np.where((lower_inner_y > upper_inner_y).sum(axis=1) == 3)[0]
    half = (lower_inner_y[flip] - upper_inner_y[flip]) * 0.5
    pts3d[flip[:, None], UPPER_INNER, 1] += half
    pts3d[flip[:, None], LOWER_INNER, 1] -= half
    if len(flip):
        pts3d[flip[:, None], UPPER_OUTER, 1] += half.mean()
        pts3d[flip[:, None], LOWER_OUTER, 1] -= half.mean()
    return pts3d


def angle2matrix(angles):
    x, y, z = np.deg2rad(angles[0]), np.deg2rad(angles[1]), np.deg2rad(angles[2])
    Rx = np.array([[1, 0, 0], [0, math.cos(x), -math.sin(x)], [0, math.sin(x), math.cos(x)]])
    Ry = np.array([[math.cos(y), 0, math.sin(y)], [0, 1, 0], [-math.sin(y), 0, math.cos(y)]])
    Rz = np.array([[math.cos(z), -math.sin(z), 0], [math.sin(z), math.cos(z), 0], [0, 0, 1]])
    return Rz.dot(Ry.dot(Rx)).astype(np.float32)


def stage5(pred_Feat, pred_Head, ident: dict, prm: dict, image_pad=None) -> dict:   # noqa: N803
    """demo.py:217-255 (``pred_Head`` is not modified).  With ``image_pad`` the shoulders get it added in fp32, as
    face_dataset.py:289-294 does before drawing.  Returns fp32 ``pred_landmarks``, ``pred_shoulders``, ``final_pts3d``
    and ``pred_headpose`` (all n_head rows, as demo.py keeps them)."""
    nframe = min(pred_Feat.shape[0], pred_Head.shape[0])
    pts = np.zeros([nframe, 73, 3])
    pts[:, MOUTH_INDICES] = pred_Feat.reshape(-1, 25, 3)[:nframe]
    if prm["Feat_smooth_sigma"] != 0:
        pts[:, 46:64] = gaussian_filter1d(pts[:, 46:64].copy().reshape(-1, 54), prm["Feat_smooth_sigma"], axis=0).reshape(-1, 18, 3)
    pts = mouth_pts_AMP(pts, True, prm["AMP_method"], prm["Feat_AMPs"])
    pts = solve_intersect_mouth(pts + ident["mean_pts3d"])
    head = pred_Head.copy()
    head[:, 0:3] *= prm["rot_AMP"]
    head[:, 3:6] *= prm["trans_AMP"]
    rs, ts = prm["Head_smooth_sigma"]
    pose = np.concatenate([gaussian_filter1d(head[:, :3], rs, axis=0), gaussian_filter1d(head[:, 3:6], ts, axis=0)],
                          axis=1).astype(np.float32)
    pose[:, 3:] += ident["mean_translation"]
    pose[:, 0] += 180
    K, scale = ident["camera_intrinsic"], np.float64(ident["scale"])
    rv, tv = np.diag([1, 1, 1]).astype(np.float32), np.zeros(3, dtype=np.float32)
    lm = np.zeros([nframe, 73, 2], dtype=np.float32)
    final = np.zeros([nframe, 73, 3], dtype=np.float32)
    final[:] = ident["std_mean_pts3d"].copy()
    final[:, 46:64] = pts[:nframe, 46:64]
    cand = ident["candidate_eye_brow"]
    for k in range(nframe):
        final[k, EYE_BROW_INDICES] = cand[k % cand.shape[0]] + ident["mean_pts3d"][EYE_BROW_INDICES]
        rot, trans = angle2matrix(pose[k][:3]), pose[k][3:][:, None]
        p = rv.dot(scale * rot.dot(final[k].T) + trans) + tv[:, None]
        p = K.dot(p)
        p[:2, :] /= p[2, :]
        lm[k] = p[:2, :].T
    sh = np.zeros([nframe, 18, 2], dtype=np.float32)
    for k in range(nframe):
        s3 = ident["shoulder3D"] + (pose[k][3:] - ident["ref_trans"]) * prm["shoulder_AMP"]
        p = K.dot(s3.astype(np.float32).T)
        p[:2, :] /= p[2, :]
        sh[k] = p[:2, :].T
    if image_pad is not None:
        top, bottom, left, right = image_pad
        sh[:, :, 0] += right - left
        sh[:, :, 1] += top - bottom
    return {"pred_landmarks": lm, "pred_shoulders": sh, "final_pts3d": final, "pred_headpose": pose}


# ------------------------------------------------------------------------------------------------------------------
# float64 truth
# ------------------------------------------------------------------------------------------------------------------
def reflect_index(i: np.ndarray, n: int) -> np.ndarray:
    """scipy.ndimage mode='reflect' (d c b a | a b c d | d c b a): period 2n."""
    m = np.mod(i, 2 * n)
    return np.where(m < n, m, 2 * n - 1 - m)


def gauss_reflect(x: np.ndarray, sigma: float) -> np.ndarray:
    """gaussian_filter1d(x, sigma, axis=0) (truncate 4, mode 'reflect') as a direct float64 sum."""
    r = int(4.0 * sigma + 0.5)
    k = np.arange(-r, r + 1)
    w = np.exp(-0.5 / (sigma * sigma) * k.astype(np.float64) ** 2)
    w /= w.sum()
    n = x.shape[0]
    out = np.zeros(x.shape)
    for j in range(2 * r + 1):
        out += w[j] * x[reflect_index(np.arange(n) + k[j], n)]
    return out


def _rotation(rad: np.ndarray) -> np.ndarray:
    """Rz Ry Rx for angles [n, 3] in radians: [n, 3, 3]."""
    cx, cy, cz = np.cos(rad[:, 0]), np.cos(rad[:, 1]), np.cos(rad[:, 2])
    sx, sy, sz = np.sin(rad[:, 0]), np.sin(rad[:, 1]), np.sin(rad[:, 2])
    o, z = np.ones_like(cx), np.zeros_like(cx)
    Rx = np.stack([o, z, z, z, cx, -sx, z, sx, cx], 1).reshape(-1, 3, 3)
    Ry = np.stack([cy, z, sy, z, o, z, -sy, z, cy], 1).reshape(-1, 3, 3)
    Rz = np.stack([cz, -sz, z, sz, cz, z, z, z, o], 1).reshape(-1, 3, 3)
    return Rz @ (Ry @ Rx)


def _mouth(feat, nframe, prm, ident, mutation=None):
    off = 18 if mutation == "mouth_shift" else 21
    x = feat[:nframe, off:off + 54].astype(np.float64)
    s = prm["Feat_smooth_sigma"]
    sm, gabs = (gauss_reflect(x, s), gauss_reflect(np.abs(x), s)) if s != 0 else (x, np.abs(x))
    amp = _amp_table(prm["AMP_method"], prm["Feat_AMPs"]).reshape(54)
    m = (sm * amp + np.asarray(ident["mean_pts3d"], np.float64)[46:64].reshape(54)).reshape(-1, 18, 3)
    lo, up = m[:, [r - 46 for r in LOWER_INNER], 1], m[:, [r - 46 for r in UPPER_INNER], 1]
    need = 2 if mutation == "lipfix_two" else 3
    flip = (lo > up).sum(axis=1) >= need
    half = np.where(flip[:, None], (lo - up) * 0.5, 0.0)
    shift = half.sum() / (3 * flip.sum()) if flip.any() else 0.0
    if mutation != "no_lipfix":
        m[:, [r - 46 for r in UPPER_INNER], 1] += half
        m[:, [r - 46 for r in LOWER_INNER], 1] -= half
        m[:, [r - 46 for r in UPPER_OUTER], 1] += np.where(flip, shift, 0.0)[:, None]
        m[:, [r - 46 for r in LOWER_OUTER], 1] -= np.where(flip, shift, 0.0)[:, None]
    noise = (2 * int(4 * s + 0.5) + 3 * int(flip.sum()) + 12) * U64 * (
        np.abs(amp) * gabs + np.abs(np.asarray(ident["mean_pts3d"], np.float64)[46:64].reshape(54)) + 2 * np.abs(half).max(initial=0.0))
    return m, flip, noise.reshape(-1, 18, 3)


def _amp_table(method, paras):
    return mouth_pts_AMP(np.ones((1, 73, 3)), True, method, paras)[0, 46:64]


def _head(head, nframe, prm, mutation=None):
    h = head[:, :6].astype(np.float64) * np.array([prm["rot_AMP"]] * 3 + [prm["trans_AMP"]] * 3, np.float64)
    if mutation == "head_nframe":
        h = h[:nframe]
    rs, ts = prm["Head_smooth_sigma"]
    if mutation == "sigma_swap":
        rs, ts = ts, rs
    s = np.concatenate([gauss_reflect(h[:, :3], rs), gauss_reflect(h[:, 3:], ts)], 1)[:nframe]
    gabs = np.concatenate([gauss_reflect(np.abs(h[:, :3]), rs), gauss_reflect(np.abs(h[:, 3:]), ts)], 1)[:nframe]
    radius = np.array([int(4 * rs + 0.5)] * 3 + [int(4 * ts + 0.5)] * 3)
    return s, gabs, radius


def truth(pred_feat, pred_head, ident: dict, prm: dict, image_pad=None) -> dict:
    """Stage 5 in float64 without intermediate roundings: ``landmarks`` [n, 73, 2], ``shoulders`` [n, 18, 2],
    ``final_pts3d`` [n, 73, 3], ``pred_headpose`` [n, 6], plus what ``error_bound`` needs."""
    n = min(pred_feat.shape[0], pred_head.shape[0])
    mouth, flip, mnoise = _mouth(pred_feat, n, prm, ident)
    s, gabs, radius = _head(pred_head, n, prm)
    pose = s + np.concatenate([[180.0, 0, 0], np.asarray(ident["mean_translation"], np.float64)])
    mean = np.asarray(ident["mean_pts3d"], np.float64)
    pts = np.broadcast_to(np.asarray(ident["std_mean_pts3d"], np.float64), (n, 73, 3)).copy()
    pts[:, 46:64] = mouth
    cand = np.asarray(ident["candidate_eye_brow"], np.float64)
    pts[:, EYE_BROW_INDICES] = cand[np.arange(n) % cand.shape[0]] + mean[EYE_BROW_INDICES]
    R = _rotation(np.deg2rad(pose[:, :3]))
    K = np.asarray(ident["camera_intrinsic"], np.float64)
    scale = float(ident["scale"])
    X = scale * np.einsum("nij,npj->npi", R, pts) + pose[:, None, 3:]
    V = X                                                   # utils.camera(): identity rotation, zero translation
    P = np.einsum("ij,npj->npi", K, V)
    lm = P[..., :2] / P[..., 2:]
    d = pose[:, 3:] - np.asarray(ident["ref_trans"], np.float64)
    s3 = np.asarray(ident["shoulder3D"], np.float64)[None] + d[:, None, :] * float(prm["shoulder_AMP"])
    Ps = np.einsum("ij,npj->npi", K, s3)
    sh = Ps[..., :2] / Ps[..., 2:]
    pad = _pad_xy(image_pad)
    return {"landmarks": lm, "shoulders": sh + pad, "final_pts3d": pts, "pred_headpose": pose, "R": R, "V": V, "P": P,
            "s": s, "gabs": gabs, "radius": radius, "mouth_noise": mnoise, "d": d, "s3": s3, "Ps": Ps,
            "sh_nopad": sh, "pad": pad, "K": K, "scale": scale, "prm": prm, "flip": flip}


def _pad_xy(image_pad) -> np.ndarray:
    if image_pad is None:
        return np.zeros(2)
    top, bottom, left, right = image_pad
    return np.array([right - left, top - bottom], np.float64)


# ------------------------------------------------------------------------------------------------------------------
# The bound
# ------------------------------------------------------------------------------------------------------------------
DEG2RAD32 = float(np.deg2rad(np.float32(1.0)))          # numpy's fp32 pi / 180


def error_bound(t: dict) -> dict:
    """Per-element bounds on |kernel - truth| for ``landmarks``, ``shoulders``, ``final_pts3d`` and ``pred_headpose``,
    first order in the roundings of csrc/lspl.cu (u = 2^-24 for fp32, e = 2^-53 for fp64), each term evaluated at the
    truth's values:

    * pose: the fp64 smoothing of h * AMP over 2r + 1 taps plus the AMP product rounds at most 2r + 3 times, each
      within e of the sum of |terms| <= gauss(|h AMP|); rounding the sum to fp32 adds u |s|, and the fp32 addition of
      mean_translation or 180 adds u |pose|.
    * final_pts3d: the fp32 store adds u |p|.  Mouth rows carry fp64 error: 2r + 1 taps, the AMP product, the mean face
      and the lip fix, whose clip mean sums 3F halves, each rounding within e of |AMP| gauss(|x|) + |mean| + 2 max|half|.
    * R: the angle picks up (pi / 180) e_pose, |a| |fp32(pi / 180) - pi / 180| and u |rad| (numpy's fp32 deg2rad);
      each entry of R moves by at most the sum of the angle errors (|dR/dangle| <= 1), plus 16 e for fp64 sin, cos and
      products (entries <= 1), plus u |R| for the fp32 rounding.
    * X = scale R p + t: sum_j (e_R |p_j| + |R| e_p_j), times scale, plus e_pose of t; V = X (identity viewpoint).
    * landmark u = P_a / P_2, P = K V: first order (K_a - u K_2) dV / P_2, so sum_j |K_aj - u K_2j| e_V_j / |P_2|, plus
      u |u| for the fp32 output.  The fp64 products, the division and every second-order product of the terms above
      stay below 2^-36 (|u| + sum_j |K_aj - u K_2j| |V_j| / |P_2|).
    * shoulders: d = t - ref_trans in fp32 adds u |d| to e_pose; the fp32 product with fp32(AMP) adds
      |fp32(AMP) - AMP| |d| + u |d AMP|; the shoulder sum adds u |s|; P = K s with two fp32 additions of three fp32
      products is within gamma_3 sum_j |K_aj| |s_j| (gamma_3 = 3u / (1 - 3u)) of K s; the fp32 division adds u |u| and
      image_pad's fp32 addition u |u + pad|.
    """
    prm = t["prm"]
    pose, s = t["pred_headpose"], t["s"]
    e_pose = U32 * (np.abs(s) + np.abs(pose)) + (2 * t["radius"] + 3) * U64 * t["gabs"]
    pts = t["final_pts3d"]
    e_p = U32 * np.abs(pts)
    e_p[:, 46:64] += t["mouth_noise"]
    rad = np.deg2rad(pose[:, :3])
    e_rad = (np.pi / 180) * e_pose[:, :3] + np.abs(pose[:, :3]) * abs(DEG2RAD32 - np.pi / 180) + U32 * np.abs(rad)
    R = t["R"]
    e_R = U32 * np.abs(R) + e_rad.sum(1)[:, None, None] + 16 * U64
    e_Rp = np.einsum("nij,npj->npi", e_R, np.abs(pts)) + np.einsum("nij,npj->npi", np.abs(R), e_p)
    e_V = t["scale"] * e_Rp + e_pose[:, None, 3:]
    K, V, P = t["K"], t["V"], t["P"]
    lm = t["landmarks"]
    b_lm = np.empty_like(lm)
    for a in range(2):
        J = np.abs(K[a][None, None, :] - lm[..., a:a + 1] * K[2][None, None, :])     # [n, 73, 3]
        P2 = np.abs(P[..., 2])
        b_lm[..., a] = ((J * e_V).sum(-1) / P2 + U32 * np.abs(lm[..., a])
                        + 2.0 ** -36 * (np.abs(lm[..., a]) + (J * np.abs(V)).sum(-1) / P2))
    amp = float(prm["shoulder_AMP"])
    amp32 = float(np.float32(amp))
    d = t["d"]
    e_d = e_pose[:, 3:] + U32 * np.abs(d)
    e_s = (amp32 * e_d + abs(amp32 - amp) * np.abs(d) + U32 * np.abs(d * amp))[:, None, :] + U32 * np.abs(t["s3"])
    g3 = 3 * U32 / (1 - 3 * U32)
    Ps, u = t["Ps"], t["sh_nopad"]
    e_P = np.einsum("ij,npj->npi", np.abs(K), e_s) + g3 * np.einsum("ij,npj->npi", np.abs(K), np.abs(t["s3"]))
    b_sh = np.empty_like(u)
    for a in range(2):
        b_sh[..., a] = ((e_P[..., a] + np.abs(u[..., a]) * e_P[..., 2]) / np.abs(Ps[..., 2]) + U32 * np.abs(u[..., a])
                        + U32 * np.abs(u[..., a] + t["pad"][a])
                        + 2.0 ** -36 * (np.abs(u[..., a]) + np.einsum("j,npj->np", np.abs(K[a]), np.abs(t["s3"])) / np.abs(Ps[..., 2])))
    return {"landmarks": b_lm, "shoulders": b_sh, "final_pts3d": e_p, "pred_headpose": e_pose}


# ------------------------------------------------------------------------------------------------------------------
# The kernel's arithmetic, emulated
# ------------------------------------------------------------------------------------------------------------------
MUTATIONS = ("head_nframe", "sigma_swap", "brow_shift", "mouth_shift", "no_lipfix", "lipfix_two", "pad_flip")


def emulate(pred_feat, pred_head, ident: dict, prm: dict, image_pad=None, mutation: Optional[str] = None) -> dict:
    """csrc/lspl.cu's steps: fp64 mouth and smoothing, fp32 pose, fp32 deg2rad, fp64 R rounded to fp32, fp32
    final_pts3d, the face projected in fp64 from fp32 values, the shoulders in fp32.  ``mutation`` (one of
    ``MUTATIONS``) plants a defect."""
    f32 = np.float32
    n = min(pred_feat.shape[0], pred_head.shape[0])
    mouth, _, _ = _mouth(pred_feat, n, prm, ident, mutation)
    s, _, _ = _head(pred_head, n, prm, mutation)
    pose = s.astype(f32)
    pose[:, 3:] += np.asarray(ident["mean_translation"], f32)
    pose[:, 0] += f32(180)
    mean = np.asarray(ident["mean_pts3d"], np.float64)
    pts = np.broadcast_to(np.asarray(ident["std_mean_pts3d"], np.float64).astype(f32), (n, 73, 3)).copy()
    pts[:, 46:64] = mouth.astype(f32)
    cand = np.asarray(ident["candidate_eye_brow"], np.float64)
    k = np.arange(n) + (1 if mutation == "brow_shift" else 0)
    pts[:, EYE_BROW_INDICES] = (cand[k % cand.shape[0]] + mean[EYE_BROW_INDICES]).astype(f32)
    rad = (pose[:, :3] * f32(DEG2RAD32)).astype(f32)
    R = _rotation(rad.astype(np.float64)).astype(f32).astype(np.float64)
    K = np.asarray(ident["camera_intrinsic"], f32)
    X = float(ident["scale"]) * np.einsum("nij,npj->npi", R, pts.astype(np.float64)) + pose[:, None, 3:].astype(np.float64)
    P = np.einsum("ij,npj->npi", K.astype(np.float64), X)
    lm = (P[..., :2] / P[..., 2:]).astype(f32)
    d = (pose[:, 3:] - np.asarray(ident["ref_trans"], f32)) * f32(prm["shoulder_AMP"])
    s3 = (np.asarray(ident["shoulder3D"], np.float64)[None] + d[:, None, :].astype(np.float64)).astype(f32)
    Ps = np.zeros(s3.shape, f32)
    for i in range(3):
        Ps[..., i] = (K[i, 0] * s3[..., 0] + K[i, 1] * s3[..., 1]) + K[i, 2] * s3[..., 2]
    sh = Ps[..., :2] / Ps[..., 2:]
    pad = _pad_xy(image_pad).astype(f32)
    if mutation == "pad_flip":
        pad = -pad
    if image_pad is not None:
        sh = sh + pad
    return {"landmarks": lm, "shoulders": sh, "final_pts3d": pts, "pred_headpose": pose}


# ------------------------------------------------------------------------------------------------------------------
# The unmodified reference (only where its checkout exists)
# ------------------------------------------------------------------------------------------------------------------
def reference_available() -> bool:
    return os.path.isfile(UTILS_FILE) and os.path.isfile(DEMO_FILE)


def reference_functions() -> types.SimpleNamespace:
    """funcs/utils.py's ``camera``, ``angle2matrix``, ``project_landmarks``, ``landmark_smooth_3d``, ``mouth_pts_AMP``,
    ``solve_intersect_mouth`` and ``headpose_smooth`` with the module-level lip index lists, lifted out with ``ast``
    and executed unchanged (the module itself imports librosa, sklearn and tqdm, so it is not imported)."""
    wanted = ("camera", "angle2matrix", "project_landmarks", "landmark_smooth_3d", "mouth_pts_AMP",
              "solve_intersect_mouth", "headpose_smooth")
    lists = ("mouth_indices", "upper_outer_lip", "upper_inner_lip", "lower_inner_lip", "lower_outer_lip", "lower_mouth",
             "upper_mouth")
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", SyntaxWarning)
        tree = ast.parse(open(UTILS_FILE).read())
    nodes = [nd for nd in tree.body
             if (isinstance(nd, (ast.FunctionDef, ast.ClassDef)) and nd.name in wanted)
             or (isinstance(nd, ast.Assign) and len(nd.targets) == 1 and getattr(nd.targets[0], "id", None) in lists)]
    assert len(nodes) == len(wanted) + len(lists), [getattr(nd, "name", None) for nd in nodes]
    ns = {"np": np, "cos": math.cos, "sin": math.sin, "gaussian_filter1d": gaussian_filter1d, "tqdm": lambda it, **kw: it}
    exec(compile(ast.fix_missing_locations(ast.Module(body=nodes, type_ignores=[])), UTILS_FILE, "exec"), ns)
    return types.SimpleNamespace(**{k: ns[k] for k in wanted})


def reference_stage5(pred_Feat, pred_Head, ident: dict, prm: dict) -> dict:   # noqa: N803
    """demo.py's statements between its ``#### 5.`` and ``#### 6.`` markers, lifted out of the ``__main__`` block with
    ``ast`` and executed unchanged on these inputs with ``reference_functions()`` as ``utils``."""
    src = open(DEMO_FILE).read()
    lines = src.splitlines()
    lo = next(i for i, ln in enumerate(lines, 1) if ln.strip().startswith("#### 5."))
    hi = next(i for i, ln in enumerate(lines, 1) if ln.strip().startswith("#### 6."))
    main = next(nd for nd in ast.parse(src).body if isinstance(nd, ast.If))
    body = [nd for nd in main.body if lo < nd.lineno < hi]
    utils = reference_functions()
    ns = dict(np=np, utils=utils, tqdm=lambda it, **kw: it, print=lambda *a, **k: None,
              mouth_indices=MOUTH_INDICES, eye_brow_indices=EYE_BROW_INDICES, camera=utils.camera(),
              pred_Feat=pred_Feat.copy(), pred_Head=pred_Head.copy(), **ident, **prm)
    exec(compile(ast.fix_missing_locations(ast.Module(body=body, type_ignores=[])), DEMO_FILE, "exec"), ns)
    return {k: ns[k] for k in ("pred_landmarks", "pred_shoulders", "final_pts3d", "pred_headpose")}
