"""APC manifold projection on the GPU (SURVEY.md 8f, row N5): drop-ins for ``KNN_with_torch`` and
``compute_LLE_projection_all_frame`` (funcs/utils.py:100-116, :171-179), stage 2 of ``demo.py`` (:196-200).

The reference computes the full [n, N] fp32 distance matrix on the host (its ``.cuda()`` calls are commented out, so this
runs on the CPU even with ``--device cuda``) and then solves one (K-1)x(K-1) normal-equation system per feature row in a
Python loop.  ``ManifoldProjector`` runs both on the device (include/lspm.h, csrc/lspm.cu): a fused distance + top-K
kernel, a merge kernel, and one warp per row solving the LLE system in fp64.  Its three calls are enqueued on the current
stream without a host synchronisation, so the projected features can go straight into ``HeadposeGenerator.generate``.

``install()`` patches the two functions of the reference's ``funcs.utils`` module; ``demo.py`` calls them as module
attributes, so it then runs unchanged.  There is no CPU path.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import numpy as np
import torch

from . import _lib

MAX_K = 32
STATUS_OK, STATUS_SINGULAR, STATUS_BAD_INDEX = 0, 1, 2


class ManifoldProjector:
    """Owns the native handle and the device copy of one feature base ``database`` [N, dim] (fp32; dim a multiple of 32,
    at most 1024).  The copy is taken at construction: later edits to the caller's array are not seen."""

    def __init__(self, database, device: Optional[torch.device] = None):
        self._lib = _lib.load()
        self._handle = C.c_void_p()
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("livespeechportraits_b200 has no CPU path: the manifold projection needs an H100 (sm_90) device")
        self.device = device if device.index is not None else torch.device("cuda", torch.cuda.current_device())
        if isinstance(database, torch.Tensor):
            database = database.detach().cpu().numpy()
        db = np.ascontiguousarray(database, dtype=np.float32)
        if db.ndim != 2:
            raise ValueError(f"database must be [N, dim], got shape {db.shape}")
        self.n_rows, self.dim = db.shape
        _lib.check_m(self._lib.lspm_create(C.byref(self._handle), int(self.dim), self.device.index))
        _lib.check_m(self._lib.lspm_load_database(self._handle, db.ctypes.data, int(self.n_rows)))

    def _feats(self, feats) -> torch.Tensor:
        f = torch.as_tensor(feats).to(device=self.device, dtype=torch.float32).contiguous()
        if f.dim() != 2 or f.shape[1] != self.dim:
            raise ValueError(f"feats must be [n, {self.dim}], got {tuple(f.shape)}")
        if f.shape[0] < 1:
            raise ValueError("feats has no rows")
        if f.data_ptr() % 16:
            f = f.clone()
        return f

    def knn(self, feats, k: int) -> torch.Tensor:
        """``KNN_with_torch`` on the device: int64 [n, k], ascending in ``|q|^2 + |d|^2 - 2 q.d`` (fp32), ties to the
        lower row.  1 <= k <= min(32, N)."""
        f = self._feats(feats)
        n = f.shape[0]
        k = int(k)
        if not 1 <= k <= min(MAX_K, self.n_rows):
            raise ValueError(f"k must be in [1, {min(MAX_K, self.n_rows)}] (got {k})")
        need = C.c_size_t()
        _lib.check_m(self._lib.lspm_workspace_bytes(self._handle, n, k, C.byref(need)))
        ws = torch.empty(max(1, need.value), dtype=torch.uint8, device=self.device)
        ind = torch.empty((n, k), dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device).cuda_stream
            _lib.check_m(self._lib.lspm_knn(self._handle, f.data_ptr(), n, k, ind.data_ptr(), None, ws.data_ptr(),
                                            need.value, stream))
        return ind

    def project(self, feats, ind, percent: float = 1.0) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
        """``compute_LLE_projection_all_frame`` and the blend of demo.py:200 on the device, given the neighbour rows
        ``ind`` [n, K] (1 <= K <= 32).  Returns ``(w, fuse, blend, status)``: float64 [n, K], fp32 [n, dim], fp32 [n, dim],
        int32 [n] (0 ok, 1 singular system, 2 an index outside [0, N); such rows hold NaN)."""
        f = self._feats(feats)
        n = f.shape[0]
        ix = torch.as_tensor(ind).to(device=self.device, dtype=torch.int64).contiguous()
        if ix.dim() != 2 or ix.shape[0] != n:
            raise ValueError(f"ind must be [{n}, K], got {tuple(ix.shape)}")
        k = ix.shape[1]
        if not 1 <= k <= MAX_K:
            raise ValueError(f"K must be in [1, {MAX_K}] (got {k})")
        w = torch.empty((n, k), dtype=torch.float64, device=self.device)
        fuse = torch.empty((n, self.dim), dtype=torch.float32, device=self.device)
        blend = torch.empty((n, self.dim), dtype=torch.float32, device=self.device)
        status = torch.empty((n,), dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device).cuda_stream
            _lib.check_m(self._lib.lspm_project(self._handle, f.data_ptr(), n, ix.data_ptr(), k, float(percent), w.data_ptr(),
                                                fuse.data_ptr(), blend.data_ptr(), status.data_ptr(), stream))
        return w, fuse, blend, status

    def project_features(self, feats, k: int, percent: float = 1.0) -> torch.Tensor:
        """Stage 2 of demo.py (:196-200) in one call: the blended features [n, dim] fp32 on the device.  Rows whose system
        is singular come back as NaN (``project`` reports which)."""
        f = self._feats(feats)
        ind = self.knn(f, k)
        return self.project(f, ind, percent)[2]

    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                self._lib.lspm_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass


def _float32_array(name: str, a) -> np.ndarray:
    if not isinstance(a, np.ndarray) or a.dtype != np.float32:
        raise TypeError(f"{name} must be a float32 numpy array (APC features are float32), got "
                        f"{type(a).__name__} of {getattr(a, 'dtype', None)}")
    return a


def KNN_with_torch(feats, feat_database, K=10):   # noqa: N802 - reference name and signature
    """Replacement for funcs/utils.py ``KNN_with_torch`` (:100-116): same arguments, same result (int64 numpy [n, K])."""
    feats = _float32_array("feats", feats)
    feat_database = _float32_array("feat_database", feat_database)
    proj = ManifoldProjector(feat_database)        # uploaded on every call: nothing is cached across calls
    return proj.knn(feats, K).cpu().numpy()


def compute_LLE_projection_all_frame(feats, feat_database, ind, nframe):   # noqa: N802 - reference name and signature
    """Replacement for funcs/utils.py ``compute_LLE_projection_all_frame`` (:171-179): returns ``(w, feat_fuse)``,
    float64 [n, K] and float32 [n, dim].  ``nframe`` is ignored, as in the reference (it is recomputed from ``feats``).
    Raises ``numpy.linalg.LinAlgError`` where ``numpy.linalg.solve`` would (a singular system)."""
    feats = _float32_array("feats", feats)
    feat_database = _float32_array("feat_database", feat_database)
    ind = np.asarray(ind)
    N = feat_database.shape[0]
    if ind.ndim != 2 or ind.shape[0] != feats.shape[0] or not np.issubdtype(ind.dtype, np.integer):
        raise ValueError(f"ind must be an integer array [{feats.shape[0]}, K], got {ind.dtype} {ind.shape}")
    if ind.size and (ind.min() < -N or ind.max() >= N):
        raise IndexError(f"ind has entries outside [-{N}, {N})")
    ind = np.where(ind < 0, ind + N, ind).astype(np.int64)           # numpy's negative indexing, as feat_database[ind[i]]
    proj = ManifoldProjector(feat_database)
    w, fuse, _, status = proj.project(feats, ind, 1.0)
    status = status.cpu().numpy()
    if (status == STATUS_SINGULAR).any():
        raise np.linalg.LinAlgError(f"Singular matrix (LLE system of row {int(np.argmax(status == STATUS_SINGULAR))})")
    return w.cpu().numpy(), fuse.cpu().numpy()


def install(module_name: str = "funcs.utils") -> None:
    """Swap the reference's KNN and LLE functions for the CUDA ones; ``demo.py`` then runs unchanged (it calls them as
    ``utils.KNN_with_torch`` / ``utils.compute_LLE_projection_all_frame``, demo.py:198-199)."""
    import importlib
    mod = importlib.import_module(module_name)
    mod.KNN_with_torch = KNN_with_torch
    mod.compute_LLE_projection_all_frame = compute_LLE_projection_all_frame
