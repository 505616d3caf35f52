"""Oracle of the live landmark post-processing (``LandmarkStream``, ``lspl_run_stream``), on top of
oracle/landmark_oracle.py.

* ``live_truth``: ``landmark_oracle.truth`` with the live lip-fix rule: the outer lips of crossed frame t move by the
  running mean of half_inner_y_diff over the crossed frames <= t (``np.cumsum`` in frame order) instead of the clip
  mean.  ``landmark_oracle.error_bound`` applies unchanged: the running sum adds at most the clip's count of terms.
* ``emulate_live``: the stream's steps in float64 with the kernel's fp32 roundings, push by push, with named defects
  (``LIVE_MUTATIONS``) that the bound must catch.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np

from oracle import landmark_oracle as O

LIVE_MUTATIONS = ("clip_mean", "exclusive_mean", "local_brow", "head_received")


def _radii(prm) -> Tuple[int, int]:
    r = lambda s: int(4.0 * float(s) + 0.5)                       # noqa: E731
    rm = r(prm["Feat_smooth_sigma"]) if prm["Feat_smooth_sigma"] != 0 else 0
    return rm, max(r(s) for s in prm["Head_smooth_sigma"])


def lip_fix_terms(pred_feat, n: int, ident: dict, prm: dict):
    """The mouth rows before the lip fix (float64 [n, 18, 3]), the crossed frames and the three half-differences."""
    m, _, _ = O._mouth(pred_feat, n, prm, ident, "no_lipfix")
    lo, up = m[:, [r - 46 for r in O.LOWER_INNER], 1], m[:, [r - 46 for r in O.UPPER_INNER], 1]
    flip = (lo > up).sum(axis=1) == 3
    half = np.where(flip[:, None], (lo - up) * 0.5, 0.0)
    return m, flip, half


def running_shift(flip: np.ndarray, half: np.ndarray, exclusive: bool = False) -> np.ndarray:
    """shift_t = S_t / (3 C_t) over the crossed frames <= t (``exclusive``: < t), 0 before the first one."""
    s, c = np.cumsum(half.sum(axis=1)), np.cumsum(flip.astype(np.int64))
    if exclusive:
        s, c = np.concatenate([[0.0], s[:-1]]), np.concatenate([[0], c[:-1]])
    return np.where(c > 0, s / (3.0 * np.maximum(c, 1)), 0.0)


def clip_shift(flip: np.ndarray, half: np.ndarray) -> float:
    return half.sum() / (3 * flip.sum()) if flip.any() else 0.0


def _outer(shift_per_frame: np.ndarray, flip: np.ndarray) -> np.ndarray:
    """[n, 18] the y offsets the outer lips of crossed frames get from a per-frame shift."""
    d = np.zeros((flip.shape[0], 18))
    d[:, [r - 46 for r in O.UPPER_OUTER]] = np.where(flip, shift_per_frame, 0.0)[:, None]
    d[:, [r - 46 for r in O.LOWER_OUTER]] = -np.where(flip, shift_per_frame, 0.0)[:, None]
    return d


def live_truth(pred_feat, pred_head, ident: dict, prm: dict, image_pad=None) -> dict:
    """``landmark_oracle.truth`` under the live lip-fix rule, plus ``shift`` (the running shift per frame),
    ``clip_shift`` and ``outer`` ([n, 73] True on the points the rule moves: rows 47-51 and 53-57 of crossed frames)."""
    t = O.truth(pred_feat, pred_head, ident, prm, image_pad)
    n = t["landmarks"].shape[0]
    _, flip, half = lip_fix_terms(pred_feat, n, ident, prm)
    run, clip = running_shift(flip, half), clip_shift(flip, half)
    pts = t["final_pts3d"].copy()
    pts[:, 46:64, 1] += _outer(run, flip) - _outer(np.full(n, clip), flip)
    X = t["scale"] * np.einsum("nij,npj->npi", t["R"], pts) + t["pred_headpose"][:, None, 3:]
    P = np.einsum("ij,npj->npi", t["K"], X)
    outer = np.zeros((n, 73), bool)
    outer[:, O.UPPER_OUTER + O.LOWER_OUTER] = flip[:, None]
    t.update(final_pts3d=pts, V=X, P=P, landmarks=P[..., :2] / P[..., 2:], shift=run, clip_shift=clip, outer=outer)
    return t


def _project(mouth, brow_index, pose, ident, prm, image_pad):
    """csrc/lspl.cu's projection of fp64 mouth rows [n, 18, 3] and fp32 poses [n, 6] (as ``landmark_oracle.emulate``)."""
    f32 = np.float32
    n = mouth.shape[0]
    mean = np.asarray(ident["mean_pts3d"], np.float64)
    pts = np.broadcast_to(np.asarray(ident["std_mean_pts3d"], np.float64).astype(f32), (n, 73, 3)).copy()
    pts[:, 46:64] = mouth.astype(f32)
    cand = np.asarray(ident["candidate_eye_brow"], np.float64)
    pts[:, O.EYE_BROW_INDICES] = (cand[brow_index % cand.shape[0]] + mean[O.EYE_BROW_INDICES]).astype(f32)
    rad = (pose[:, :3] * f32(O.DEG2RAD32)).astype(f32)
    R = O._rotation(rad.astype(np.float64)).astype(f32).astype(np.float64)
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
    if image_pad is not None:
        sh = sh + O._pad_xy(image_pad).astype(f32)
    return {"landmarks": lm, "shoulders": sh, "final_pts3d": pts, "pred_headpose": pose}


def _pose(head, n_reflect, frames, prm, ident):
    f32 = np.float32
    s, _, _ = O._head(head[:n_reflect], n_reflect, prm)
    pose = s[frames].astype(f32)
    pose[:, 3:] += np.asarray(ident["mean_translation"], f32)
    pose[:, 0] += f32(180)
    return pose


def emulate_live(pred_feat, pred_head, ident: dict, prm: dict, pushes: Sequence[Tuple[int, int]], image_pad=None,
                 mutation: Optional[str] = None) -> dict:
    """The live path pushed as (mouth rows, head rows) pieces, then finished: each push emits the frames
    ``stream.landmark_counts`` allows and computes them with the kernel's arithmetic.  ``mutation``:
    ``clip_mean`` (the clip's mean shift), ``exclusive_mean`` (the running mean without frame t), ``local_brow``
    (eyebrow candidate from the push's local frame index), ``head_received`` (a stream that forgets the head-pose
    look-ahead: it emits by the mouth rule alone and reflects the head at the rows received)."""
    from livespeechportraits_b200.stream import landmark_counts
    n = min(pred_feat.shape[0], pred_head.shape[0])
    rm, rh = _radii(prm)
    m, flip, half = lip_fix_terms(pred_feat, n, ident, prm)
    shift = (np.full(n, clip_shift(flip, half)) if mutation == "clip_mean"
             else running_shift(flip, half, exclusive=mutation == "exclusive_mean"))
    m = m.copy()
    m[:, [r - 46 for r in O.UPPER_INNER], 1] += half
    m[:, [r - 46 for r in O.LOWER_INNER], 1] -= half
    m[:, :, 1] += _outer(shift, flip)
    parts, done, F, H = [], 0, 0, 0
    for push in list(pushes) + [None]:
        finished = push is None
        if not finished:
            F, H = min(F + push[0], pred_feat.shape[0]), min(H + push[1], pred_head.shape[0])
        if mutation == "head_received" and not finished:
            upto = max(0, min(F, H) - rm)
        else:
            upto = landmark_counts(F, H, finished, rm, rh)
        frames = np.arange(done, upto)
        if frames.size:
            n_reflect = H if mutation == "head_received" else pred_head.shape[0]
            brow = frames - done if mutation == "local_brow" else frames
            parts.append(_project(m[frames], brow, _pose(pred_head, n_reflect, frames, prm, ident), ident, prm, image_pad))
        done = upto
    keys = ("landmarks", "shoulders", "final_pts3d", "pred_headpose")
    if not parts:
        return {k: np.zeros((0,) + s, np.float32) for k, s in zip(keys, ((73, 2), (18, 2), (73, 3), (6,)))}
    return {k: np.concatenate([p[k] for p in parts]) for k in keys}
