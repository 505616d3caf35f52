"""Landmark post-processing on the GPU (SURVEY.md 8f, row N7): stage 5 of ``demo.py`` (:215-255).

The reference takes the mouth track of Audio2Feature and the head-pose track of Audio2Headpose back to the host, smooths
and amplifies them in numpy (``landmark_smooth_3d``, ``mouth_pts_AMP``, ``solve_intersect_mouth``, ``headpose_smooth``)
and projects every frame in two Python loops (``project_landmarks`` for the 73 face points, then the 18 shoulder
points).  ``LandmarkPostprocessor.run`` does all of it in two kernels (include/lspl.h, csrc/lspl.cu) and leaves
``pred_landmarks`` / ``pred_shoulders`` on the device, where ``Feature2Face_G.draw_feature_maps`` and
``ClipRenderer.render_clip_from_landmarks`` take them.  ``postprocess_clip`` is the numpy-in, numpy-out form with
demo.py's variable names.  There is no CPU path.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional, Sequence

import numpy as np
import torch

from . import _lib

N_PTS = 73
N_SHOULDERS = 18
MOUTH_ROWS = range(46, 64)
UPPER_MOUTH = [46, 47, 48, 49, 50, 51, 52, 61, 62, 63]     # funcs/utils.py:273
LOWER_MOUTH = [53, 54, 55, 56, 57, 58, 59, 60]             # funcs/utils.py:272
MAX_RADIUS = 1024                                          # LSPL_MAX_RADIUS


def amp_table(method: str, paras: Sequence[float]) -> np.ndarray:
    """``mouth_pts_AMP(pts3d, is_delta=True, method, paras)`` (funcs/utils.py:274-325) as one scale per (mouth row 46 + i,
    coordinate): float64 [18, 3].  Multiplying rows 46..63 by it gives the reference's result bit for bit.  ``delta`` and
    ``CloseSmall`` (no shipped config uses them; ``CloseSmall`` decides per frame) raise ``NotImplementedError``; any
    other name raises ``ValueError``."""
    paras = [float(p) for p in paras]
    table = np.ones((18, 3), np.float64)
    if method in ("XY", "XYZ"):
        if len(paras) != len(method):
            raise ValueError(f"AMP method {method!r} takes {len(method)} factors, got {len(paras)}")
        table[:, :len(paras)] = paras
    elif method == "LowerMore":
        if len(paras) != 6:
            raise ValueError(f"AMP method 'LowerMore' takes 6 factors, got {len(paras)}")
        table[[r - 46 for r in UPPER_MOUTH]] = paras[:3]
        table[[r - 46 for r in LOWER_MOUTH]] = paras[3:]
    elif method in ("delta", "CloseSmall"):
        raise NotImplementedError(f"AMP method {method!r} is not supported on the device (no shipped config uses it)")
    else:
        raise ValueError(f"unknown AMP method {method!r}: expected 'XY', 'XYZ' or 'LowerMore'")
    return table


@dataclass
class Identity:
    """The constants demo.py loads once per identity (:81-108).  ``camera_intrinsic``, ``mean_translation`` and
    ``ref_trans`` hold fp32 values in the reference; ``relative_rotation`` / ``relative_translation`` are
    ``utils.camera()``'s (identity and zero)."""
    mean_pts3d: np.ndarray            # [73, 3]
    std_mean_pts3d: np.ndarray        # [73, 3]
    candidate_eye_brow: np.ndarray    # [m, 16, 3]
    mean_translation: np.ndarray      # [3]
    ref_trans: np.ndarray             # [3]
    shoulder3D: np.ndarray            # [18, 3]
    camera_intrinsic: np.ndarray      # [3, 3]
    scale: float
    relative_rotation: Optional[np.ndarray] = None      # [3, 3], default identity
    relative_translation: Optional[np.ndarray] = None   # [3], default zero


@dataclass
class StageParams:
    """The per-identity settings of config/<id>.yaml that stage 5 reads (demo.py:120-126)."""
    feat_smooth_sigma: float          # Audio2Mouth smooth (0: no smoothing)
    amp_method: str                   # Audio2Mouth AMP[0]
    feat_amps: Sequence[float]        # Audio2Mouth AMP[1:]
    rot_amp: float                    # Headpose AMP
    trans_amp: float
    head_smooth_sigma: Sequence[float]   # Headpose smooth: (rot, trans), both > 0
    shoulder_amp: float


def _f64(a, shape) -> np.ndarray:
    a = np.ascontiguousarray(np.asarray(a, dtype=np.float64))
    if a.shape != shape:
        raise ValueError(f"expected shape {shape}, got {a.shape}")
    return a


def _native_params(p: StageParams, image_pad) -> _lib.LsplParams:
    rot_sigma, trans_sigma = (float(s) for s in p.head_smooth_sigma)
    for name, s in (("rot", rot_sigma), ("trans", trans_sigma)):
        if not s > 0:
            raise ValueError(f"head {name} smoothing sigma must be > 0 (got {s}): scipy's gaussian_filter1d divides by zero")
    feat_sigma = float(p.feat_smooth_sigma)
    if not feat_sigma >= 0:
        raise ValueError(f"mouth smoothing sigma must be >= 0 (got {feat_sigma})")
    for s in (feat_sigma, rot_sigma, trans_sigma):
        if int(4.0 * s + 0.5) > MAX_RADIUS:
            raise ValueError(f"smoothing sigma {s} has a radius above {MAX_RADIUS}")
    n = _lib.LsplParams()
    n.feat_sigma, n.rot_sigma, n.trans_sigma = feat_sigma, rot_sigma, trans_sigma
    table = amp_table(p.amp_method, p.feat_amps)
    for i in range(18):
        for c in range(3):
            n.amp[i][c] = table[i, c]
    n.rot_amp, n.trans_amp, n.shoulder_amp = float(p.rot_amp), float(p.trans_amp), float(p.shoulder_amp)
    if image_pad is not None:
        n.use_pad = 1
        for i, v in enumerate(image_pad):
            n.pad[i] = int(v)
    return n


class LandmarkPostprocessor:
    """Owns the native handle and the device copy of one identity's constants (taken at construction)."""

    def __init__(self, identity: Identity, device: Optional[torch.device] = None):
        self._lib = _lib.load()
        self._handle = C.c_void_p()
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("livespeechportraits_b200 has no CPU path: the landmark post-processing needs an H100 (sm_90) device")
        self.device = device if device.index is not None else torch.device("cuda", torch.cuda.current_device())
        cand = np.ascontiguousarray(np.asarray(identity.candidate_eye_brow, dtype=np.float64))
        if cand.ndim != 3 or cand.shape[1:] != (16, 3) or cand.shape[0] < 1:
            raise ValueError(f"candidate_eye_brow must be [m >= 1, 16, 3], got {cand.shape}")
        rv = np.eye(3) if identity.relative_rotation is None else identity.relative_rotation
        tv = np.zeros(3) if identity.relative_translation is None else identity.relative_translation
        self._keep = [_f64(identity.mean_pts3d, (N_PTS, 3)), _f64(identity.std_mean_pts3d, (N_PTS, 3)), cand,
                      _f64(identity.shoulder3D, (N_SHOULDERS, 3))]
        nid = _lib.LsplIdentity()
        nid.mean_pts3d, nid.std_mean_pts3d, nid.candidate_eye_brow, nid.shoulder3D = (a.ctypes.data for a in self._keep)
        nid.n_candidates = cand.shape[0]
        nid.mean_translation[:] = _f64(identity.mean_translation, (3,)).tolist()
        nid.ref_trans[:] = _f64(identity.ref_trans, (3,)).tolist()
        nid.camera_intrinsic[:] = _f64(identity.camera_intrinsic, (3, 3)).ravel().tolist()
        nid.relative_rotation[:] = _f64(rv, (3, 3)).ravel().tolist()
        nid.relative_translation[:] = _f64(tv, (3,)).tolist()
        nid.scale = float(identity.scale)
        _lib.check_l(self._lib.lspl_create(C.byref(self._handle), self.device.index))
        _lib.check_l(self._lib.lspl_load_identity(self._handle, C.byref(nid)))
        del self._keep

    def run(self, pred_feat, pred_head, params: StageParams, image_pad: Optional[Sequence[int]] = None,
            return_intermediates: bool = False):
        """Stage 5 for ``nframe = min(n_feat, n_head)`` frames.  ``pred_feat`` [n_feat, 75] (or [n_feat, 25, 3]) and
        ``pred_head`` [n_head, >= 6]: numpy or torch, rounded to fp32 (the network outputs they come from are fp32).
        ``image_pad`` (top, bottom, left, right) is added to the shoulders as face_dataset.py's get_feature_image does.
        Returns CUDA fp32 ``landmarks`` [nframe, 73, 2] and ``shoulders`` [nframe, 18, 2], and with
        ``return_intermediates`` also ``final_pts3d`` [nframe, 73, 3] and ``pred_headpose`` [nframe, 6] (demo.py's
        values of those names).  Enqueued on the current stream; no host synchronisation for device inputs."""
        native = _native_params(params, image_pad)
        dev = self.device
        feat = torch.as_tensor(pred_feat).to(device=dev, dtype=torch.float32)
        head = torch.as_tensor(pred_head).to(device=dev, dtype=torch.float32)
        if feat.numel() % 75 or (feat.dim() == 3 and tuple(feat.shape[1:]) != (25, 3)) or feat.dim() not in (2, 3) \
                or (feat.dim() == 2 and feat.shape[1] != 75):
            raise ValueError(f"pred_feat must be [n, 75] or [n, 25, 3], got {tuple(feat.shape)}")
        feat = feat.reshape(-1, 75).contiguous()
        if head.dim() != 2 or head.shape[1] < 6:
            raise ValueError(f"pred_head must be [n, >= 6], got {tuple(head.shape)}")
        head = head.contiguous()
        n_feat, n_head = feat.shape[0], head.shape[0]
        n = min(n_feat, n_head)
        f32 = dict(dtype=torch.float32, device=dev)
        lm = torch.empty((n, N_PTS, 2), **f32)
        sh = torch.empty((n, N_SHOULDERS, 2), **f32)
        pts = torch.empty((n, N_PTS, 3), **f32) if return_intermediates else None
        pose = torch.empty((n, 6), **f32) if return_intermediates else None
        nbytes = C.c_size_t()
        _lib.check_l(self._lib.lspl_workspace_bytes(self._handle, n_feat, n_head, C.byref(nbytes)))
        ws = torch.empty((max(nbytes.value, 1),), dtype=torch.uint8, device=dev)
        ptr = lambda t: t.data_ptr() if t is not None and t.numel() else None    # noqa: E731
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check_l(self._lib.lspl_run(self._handle, ptr(feat), n_feat, ptr(head), n_head, head.shape[1], C.byref(native),
                                            ptr(lm), ptr(sh), ptr(pts), ptr(pose), ws.data_ptr(), ws.numel(), stream))
        return (lm, sh, pts, pose) if return_intermediates else (lm, sh)

    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                self._lib.lspl_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass


def postprocess_clip(pred_Feat, pred_Head, mean_pts3d, std_mean_pts3d, candidate_eye_brow, mean_translation, ref_trans,
                     shoulder3D, camera_intrinsic, scale, Feat_smooth_sigma, AMP_method, Feat_AMPs, rot_AMP, trans_AMP,
                     Head_smooth_sigma, shoulder_AMP, camera=None, device=None):   # noqa: N803 - demo.py's names
    """demo.py :217-255 with demo.py's variables: returns ``pred_landmarks`` [nframe, 73, 2] and ``pred_shoulders``
    [nframe, 18, 2] as float32 numpy.  ``camera`` is ``utils.camera()`` (its relative rotation and translation; None:
    identity and zero).  Unlike demo.py:228-229 it leaves ``pred_Head`` unchanged.  Raises ``ValueError`` for a head
    smoothing sigma of 0, where scipy raises ``ZeroDivisionError``."""
    ident = Identity(mean_pts3d, std_mean_pts3d, candidate_eye_brow, mean_translation, ref_trans, shoulder3D,
                     camera_intrinsic, scale, getattr(camera, "relative_rotation", None),
                     getattr(camera, "relative_translation", None))
    params = StageParams(Feat_smooth_sigma, AMP_method, Feat_AMPs, rot_AMP, trans_AMP, Head_smooth_sigma, shoulder_AMP)
    _native_params(params, None)                 # refuse bad settings before any device work
    lm, sh = LandmarkPostprocessor(ident, device).run(pred_Feat, pred_Head, params)
    return lm.cpu().numpy(), sh.cpu().numpy()
