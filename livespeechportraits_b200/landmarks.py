"""Landmark post-processing on the GPU (SURVEY.md 8f, row N7): stage 5 of ``demo.py`` (:215-255).

The reference takes the mouth track of Audio2Feature and the head-pose track of Audio2Headpose back to the host, smooths
and amplifies them in numpy (``landmark_smooth_3d``, ``mouth_pts_AMP``, ``solve_intersect_mouth``, ``headpose_smooth``)
and projects every frame in two Python loops (``project_landmarks`` for the 73 face points, then the 18 shoulder
points).  ``LandmarkPostprocessor.run`` does all of it in two kernels (include/lspl.h, csrc/lspl.cu) and leaves
``pred_landmarks`` / ``pred_shoulders`` on the device, where ``Feature2Face_G.draw_feature_maps`` and
``ClipRenderer.render_clip_from_landmarks`` take them.  ``postprocess_clip`` is the numpy-in, numpy-out form with
demo.py's variable names.  ``LandmarkPostprocessor.stream`` opens a ``LandmarkStream``: track rows pushed as they
arrive from ``stream.AudioStream``, landmarks out as soon as the smoothing windows are in.  There is no CPU path.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import NamedTuple, Optional, Sequence, Tuple

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


def radii(params: StageParams) -> Tuple[int, int]:
    """The look-ahead of stage 5 in frames: the mouth smoothing radius ``rm`` (0 without smoothing) and
    ``rh = max(rr, rt)`` of the two head-pose smoothings, each ``int(4 sigma + 0.5)``."""
    r = lambda s: int(4.0 * float(s) + 0.5)                       # noqa: E731
    rm = r(params.feat_smooth_sigma) if float(params.feat_smooth_sigma) > 0 else 0
    return rm, max(r(s) for s in params.head_smooth_sigma)


class LandmarkRows(NamedTuple):
    """What one ``LandmarkStream.push`` or ``finish`` returned: frames ``frame0 .. frame0 + k - 1``."""
    landmarks: torch.Tensor                        # [k, 73, 2]
    shoulders: torch.Tensor                        # [k, 18, 2]
    frame0: int
    final_pts3d: Optional[torch.Tensor] = None     # [k, 73, 3] with return_intermediates
    pred_headpose: Optional[torch.Tensor] = None   # [k, 6] with return_intermediates


class LandmarkPostprocessor(_lib.Handle):
    """Owns the native handle and the device copy of one identity's constants (taken at construction)."""
    prefix, what = "lspl", "the landmark post-processing"

    def __init__(self, identity: Identity, device: Optional[torch.device] = None):
        super().__init__(device)
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
        self._create()
        self.call("load_identity", C.byref(nid))
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
        ws = self.workspace(n_feat, n_head)
        ptr = lambda t: t.data_ptr() if t is not None and t.numel() else None    # noqa: E731
        with self.cuda_stream() as stream:
            self.call("run", ptr(feat), n_feat, ptr(head), n_head, head.shape[1], C.byref(native), ptr(lm), ptr(sh), ptr(pts),
                      ptr(pose), ws.data_ptr(), ws.numel(), stream)
        return (lm, sh, pts, pose) if return_intermediates else (lm, sh)

    def stream(self, params: StageParams, image_pad: Optional[Sequence[int]] = None,
               return_intermediates: bool = False) -> "LandmarkStream":
        """A stream over one clip's mouth and head-pose track rows (``LandmarkStream``)."""
        return LandmarkStream(self, params, image_pad, return_intermediates)

    def stream_state(self) -> torch.Tensor:
        """A device buffer for ``lspl_run_stream``'s lip-fix state (its first call, at frame 0, initialises it)."""
        if self.device is None:
            raise RuntimeError("host-only handle: created with device=-1")
        need = C.c_size_t()
        self.call("stream_state_bytes", C.byref(need))
        return torch.empty(need.value, dtype=torch.uint8, device=self.device)

    def device_rows(self, rows, width: int) -> torch.Tensor:
        """Track rows (numpy or torch, any device) as contiguous fp32 device rows of their first ``width`` columns:
        ``[n, 75]`` (or ``[n, 25, 3]``) for the mouth, ``[n, >= 6]`` for the head pose (``width`` 6)."""
        t = _lib.to_device(rows, self.device)
        t = t.reshape(-1, 75) if width == 75 and t.dim() == 3 else t
        if t.dim() != 2 or t.shape[1] < width or (width == 75 and t.shape[1] != 75):
            raise ValueError(f"track rows must be [n, {width if width == 75 else '>= 6'}], got {tuple(t.shape)}")
        return t[:, :width].contiguous()

    def run_stream(self, feat, feat_row0: int, head, head_row0: int, frame0: int, n: int, nframe_total: int,
                   n_head_total: int, native, state, ws, return_intermediates: bool):
        """One ``lspl_run_stream`` call over the device rows ``feat`` [*, 75] and ``head`` [*, 6] (fp32, contiguous):
        returns ``LandmarkRows`` of frames ``frame0 .. frame0 + n - 1`` and the workspace used (``ws`` or a larger one)."""
        dev = self.device
        f32 = dict(dtype=torch.float32, device=dev)
        lm, sh = torch.empty((n, N_PTS, 2), **f32), torch.empty((n, N_SHOULDERS, 2), **f32)
        pts = torch.empty((n, N_PTS, 3), **f32) if return_intermediates else None
        pose = torch.empty((n, 6), **f32) if return_intermediates else None
        need = C.c_size_t()
        self.call("stream_workspace_bytes", n, C.byref(need))
        ws = _lib.reserve(ws, need.value, dev)
        ptr = lambda t: t.data_ptr() if t is not None and t.numel() else None    # noqa: E731
        with self.cuda_stream() as stream:
            self.call("run_stream", ptr(feat), feat_row0, feat.shape[0], ptr(head), head_row0, head.shape[0], 6, frame0, n,
                      nframe_total, n_head_total, C.byref(native), ptr(lm), ptr(sh), ptr(pts), ptr(pose), state.data_ptr(),
                      ws.data_ptr(), ws.numel(), stream)
        return LandmarkRows(lm, sh, frame0, pts, pose), ws


class LandmarkStream:
    """Stage 5 over track rows that arrive in pieces (``LandmarkPostprocessor.stream``).  ``push(mouth_rows, head_rows)``
    takes the new rows of the Audio2Mouth track ([m, 75] or [m, 25, 3]) and of the head-pose track ([h, >= 6]), in any
    counts, and ``finish()`` ends the clip; both return ``LandmarkRows`` of the frames that became ready
    (``stream.landmark_counts``: frame t needs mouth rows up to t + rm and head rows up to t + rh; at the end every
    frame of ``nframe = min(n_feat, n_head)``).

    Every value equals ``run`` on the whole tracks bit for bit, except the outer lips of crossed frames: there
    ``solve_intersect_mouth``'s mean over all crossed frames of the clip, which a live stream cannot know, becomes the
    running mean over the crossed frames up to and including the frame (include/lspl.h, ``lspl_run_stream``).  It does
    not depend on how the rows were cut into pushes, and at the clip's last crossed frame it equals the clip mean up to
    fp64 summation order.

    Kept on the device: the mouth rows from ``frames - rm``, the head rows from ``frames - rh``, the lip-fix state (a
    running sum and count) and a workspace sized for the largest push so far.  Pushes make no host synchronisation and
    go on one CUDA stream."""

    def __init__(self, post, params: StageParams, image_pad=None, return_intermediates: bool = False):
        self._post = post
        self._native = _native_params(params, image_pad)
        self.rm, self.rh = radii(params)
        self._inter = bool(return_intermediates)
        self._state = post.stream_state()
        self._ws = None
        self._feat = post.device_rows(torch.empty((0, 75)), 75)
        self._head = post.device_rows(torch.empty((0, 6)), 6)
        self._feat_row0 = self._head_row0 = 0      # global index of the first kept row
        self.feat_rows = self.head_rows = 0        # rows pushed so far
        self.frames = 0                            # frames returned so far
        self.finished = False

    def push(self, mouth_rows, head_rows) -> LandmarkRows:
        if self.finished:
            raise RuntimeError("the stream has finished")
        feat, head = self._post.device_rows(mouth_rows, 75), self._post.device_rows(head_rows, 6)
        self._feat = torch.cat([self._feat, feat]) if feat.shape[0] else self._feat
        self._head = torch.cat([self._head, head]) if head.shape[0] else self._head
        self.feat_rows += feat.shape[0]
        self.head_rows += head.shape[0]
        return self._emit(False)

    def finish(self) -> LandmarkRows:
        if self.finished:
            raise RuntimeError("the stream has finished")
        self.finished = True
        return self._emit(True)

    def _emit(self, finished: bool) -> LandmarkRows:
        from .stream import landmark_counts
        n = landmark_counts(self.feat_rows, self.head_rows, finished, self.rm, self.rh) - self.frames
        nframe, n_head = (min(self.feat_rows, self.head_rows), self.head_rows) if finished else (-1, -1)
        out, self._ws = self._post.run_stream(self._feat, self._feat_row0, self._head, self._head_row0, self.frames, n,
                                              nframe, n_head, self._native, self._state, self._ws, self._inter)
        self.frames += n
        # keep the rows later frames read: mouth from frames - rm, head from frames - rh
        drop = min(max(self.frames - self.rm - self._feat_row0, 0), self._feat.shape[0])
        self._feat, self._feat_row0 = self._feat[drop:].clone(), self._feat_row0 + drop
        drop = min(max(self.frames - self.rh - self._head_row0, 0), self._head.shape[0])
        self._head, self._head_row0 = self._head[drop:].clone(), self._head_row0 + drop
        return out if self._inter else LandmarkRows(out.landmarks, out.shoulders, out.frame0)


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
