"""ctypes binding of the C ABI in include/lspg.h, include/lsph.h, include/lspm.h, include/lspa.h, include/lspl.h, include/lspr.h, include/lspj.h and include/lspv.h.  Plain pointers and sizes only."""
from __future__ import annotations

import contextlib
import ctypes as C
import os
from typing import List, Optional, Tuple

import torch

from . import build as _build

LSPG_VARIANT = {"normal": 0, "large": 1}
LSPG_MODE = {"fast": 0, "parity": 1}
LSPR_KIND = {"apc": 0, "mouth": 1}


class LsphConfig(C.Structure):
    _fields_ = [(k, C.c_int) for k in ("apc_hidden", "frame_future", "layers", "blocks", "residual_ch", "dilation_ch", "skip_ch",
                                       "kernel_size", "use_bias", "cond_ch", "input_ch", "ncenter", "ndim", "loss_gmm")]


class LsprConfig(C.Structure):
    _fields_ = [(k, C.c_int) for k in ("kind", "input_dim", "hidden", "num_layers", "residual", "frame_future", "out_dim")]


class LsplIdentity(C.Structure):
    _fields_ = [("mean_pts3d", C.c_void_p), ("std_mean_pts3d", C.c_void_p), ("candidate_eye_brow", C.c_void_p),
                ("n_candidates", C.c_int), ("mean_translation", C.c_double * 3), ("ref_trans", C.c_double * 3),
                ("shoulder3D", C.c_void_p), ("camera_intrinsic", C.c_double * 9), ("relative_rotation", C.c_double * 9),
                ("relative_translation", C.c_double * 3), ("scale", C.c_double)]


class LsplParams(C.Structure):
    _fields_ = [("feat_sigma", C.c_double), ("rot_sigma", C.c_double), ("trans_sigma", C.c_double),
                ("amp", (C.c_double * 3) * 18), ("rot_amp", C.c_double), ("trans_amp", C.c_double),
                ("shoulder_amp", C.c_double), ("use_pad", C.c_int), ("pad", C.c_int * 4)]


class LspgTensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.POINTER(C.c_float)), ("numel", C.c_int64)]


class LspgLayerInfo(C.Structure):
    _fields_ = [
        ("kind", C.c_int), ("n_src", C.c_int), ("src", C.c_int * 2), ("cin", C.c_int * 2),
        ("out", C.c_int), ("res", C.c_int), ("cout", C.c_int), ("cout_pad", C.c_int),
        ("n_phases", C.c_int), ("n_taps", C.c_int), ("k_total", C.c_int), ("relu", C.c_int), ("has_bn", C.c_int),
        ("tap_map", (C.c_int8 * 9) * 4), ("tap_dx", (C.c_int8 * 9) * 4), ("tap_dy", (C.c_int8 * 9) * 4),
        ("conv_key", C.c_char * 96), ("bn_key", C.c_char * 96),
    ]


class LspgLayerGeo(C.Structure):
    _fields_ = [("kernel", C.c_int), ("bn", C.c_int), ("tile_w", C.c_int), ("tile_h", C.c_int), ("tile_n", C.c_int),
                ("m_tiles", C.c_int), ("n_tiles", C.c_int), ("n_phases", C.c_int), ("n_split", C.c_int), ("split_len", C.c_int),
                ("k_items", C.c_int), ("ctas", C.c_int), ("partial_bytes", C.c_int64), ("cluster", C.c_int),
                ("w_box_taps", C.c_int * 2)]




_p, _i, _i64, _sz = C.c_void_p, C.c_int, C.c_int64, C.c_size_t      # handles, device pointers and streams are _p
_out_handle, _pi, _pi64, _psz = C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.POINTER(C.c_int64), C.POINTER(C.c_size_t)
_tensors = C.POINTER(LspgTensor)
_forward = [_p, _p, _i64, _p, _i64, _p, _i, _i, _i, _p, _sz, _i, _p]

# Every C-ABI symbol and its argument types.  restype is c_char_p for *_last_error and c_int (0 or LSPG_E*) otherwise.
ARGTYPES = {
    # include/lspg.h (Feature2Face generator and feature-map rasteriser)
    "lspg_create": [_out_handle, _i, _i, _i, _i, _i, _i],
    "lspg_load_weights": [_p, _tensors, _i],
    "lspg_workspace_bytes": [_p, _i, _i, _i, _i, _psz],
    "lspg_forward": _forward,
    "lspg_forward_image": _forward,
    "lspg_draw_feature_maps": [_p, _p, _p, _i, _p, _i, _i, _i, _p],
    "lspg_destroy": [_p],
    "lspg_last_error": [],
    "lspg_num_layers": [_p, _pi],
    "lspg_layer_info_get": [_p, _i, C.POINTER(LspgLayerInfo)],
    "lspg_layer_packed": [_p, _i, _i, _p, _i64],
    "lspg_layer_affine": [_p, _i, _p, _p, _i64],
    "lspg_num_tensors": [_p, _pi],
    "lspg_tensor_shape": [_p, _i, _i, _i, _pi, _pi, _pi],
    "lspg_debug_read_tensor": [_p, _i, _i, _p, _i64],
    "lspg_launches_per_forward": [_p, _pi],
    "lspg_flops_per_frame": [_p, _i, _i, C.POINTER(C.c_double)],
    "lspg_profile_enable": [_p, _i],
    "lspg_profile_read": [_p, _p, _i, _pi],
    "lspg_debug_read_trace": [_p, _p, _i64],
    "lspg_debug_fast_div": [C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32)],
    "lspg_debug_layer_geo": [_p, _i, _i, _i, _i, C.POINTER(LspgLayerGeo)],
    "lspg_graph_stats": [_p, _pi64, _pi64, _pi64],
    "lspg_release_workspace": [_p, _p],
    # include/lsph.h (Audio2Headpose generation loop)
    "lsph_create": [_out_handle, C.POINTER(LsphConfig), _i],
    "lsph_load_weights": [_p, _tensors, _i],
    "lsph_state_bytes": [_p, _psz],
    "lsph_stream_workspace_bytes": [_p, _i, _psz],
    "lsph_generate_stream": [_p, _p, _i, _i, _i, _i, _p, _p, _p, C.c_float, _p, _p, _p, _p, _sz, _i, _p],
    "lsph_receptive_field": [_p, _pi],
    "lsph_debug_packed": [_p, _i, _p, _i64],
    "lsph_destroy": [_p],
    "lsph_last_error": [],
    # include/lspm.h (APC manifold projection: KNN + LLE)
    "lspm_create": [_out_handle, _i, _i],
    "lspm_load_database": [_p, _p, _i64],
    "lspm_workspace_bytes": [_p, _i, _i, _psz],
    "lspm_knn": [_p, _p, _i, _i, _p, _p, _p, _sz, _p],
    "lspm_project": [_p, _p, _i, _p, _i, C.c_float, _p, _p, _p, _p, _p],
    "lspm_destroy": [_p],
    "lspm_last_error": [],
    # include/lspa.h (log-mel front end)
    "lspa_create": [_out_handle, _i],
    "lspa_load_mel_basis": [_p, _p, _i, _i],
    "lspa_logmel_at": [_p, _p, _i64, _i64, _i, _i, _i, C.c_double, _i, _p, _p],
    "lspa_load_resample_filter": [_p, _p, _p, _i, _i, C.c_double],
    "lspa_resample_at": [_p, _p, _i, _i, _i64, _i64, _i64, _i64, _p, _i, _p, _p],
    "lspa_destroy": [_p],
    "lspa_last_error": [],
    # include/lspl.h (landmark post-processing, demo.py stage 5)
    "lspl_create": [_out_handle, _i],
    "lspl_load_identity": [_p, C.POINTER(LsplIdentity)],
    "lspl_workspace_bytes": [_p, _i, _i, _psz],
    "lspl_run": [_p, _p, _i, _p, _i, _i, C.POINTER(LsplParams), _p, _p, _p, _p, _p, _sz, _p],
    "lspl_stream_state_bytes": [_p, _psz],
    "lspl_stream_workspace_bytes": [_p, _i, _psz],
    "lspl_run_stream": [_p, _p, _i, _i, _p, _i, _i, _i, _i, _i, _i, _i, C.POINTER(LsplParams), _p, _p, _p, _p, _p, _p, _sz, _p],
    "lspl_destroy": [_p],
    "lspl_last_error": [],
    # include/lspr.h (APC encoder GRU and Audio2Mouth LSTM, demo.py stages 1 and 3)
    "lspr_create": [_out_handle, C.POINTER(LsprConfig), _i],
    "lspr_load_weights": [_p, _tensors, _i],
    "lspr_workspace_bytes": [_p, _i, _psz],
    "lspr_state_bytes": [_p, _psz],
    "lspr_forward_stream": [_p, _p, _i, _i64, _p, _p, _p, _sz, _i, _p],
    "lspr_debug_packed": [_p, _i, _p, _pi64],
    "lspr_destroy": [_p],
    "lspr_last_error": [],
    # include/lspj.h (baseline JPEG encoder, demo.py's JPEG boundary)
    "lspj_create": [_out_handle, _i],
    "lspj_max_bytes": [_p, _i, _i, _i, _psz],
    "lspj_workspace_bytes": [_p, _i, _i, _i, _i, _psz],
    "lspj_encode": [_p, _p, _i, _i, _i, _i, _i, _p, _i64, _p, _p, _sz, _p],
    "lspj_destroy": [_p],
    "lspj_last_error": [],
    # include/lspv.h (H.264 Constrained Baseline encoder)
    "lspv_create": [_out_handle, _i, _i, _i, _i, _i],
    "lspv_max_bytes": [_p, _i, _i, _psz],
    "lspv_state_bytes": [_p, _i, _i, _psz],
    "lspv_workspace_bytes": [_p, _i, _i, _psz],
    "lspv_encode": [_p, _p, _i, _i, _i, _i, _i64, _p, _p, _i64, _p, _p, _p, _sz, _p],
    "lspv_destroy": [_p],
    "lspv_last_error": [],
}


def symbols(prefix: Optional[str] = None) -> List[str]:
    """The bound symbols of one module (``"lspm"``, ...), or of all eight."""
    return [name for name in ARGTYPES if prefix is None or name.startswith(prefix + "_")]


class LspgError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"lspg error {code}: {message}")
        self.code = code


_LIB: Optional[C.CDLL] = None


def library_path() -> str:
    return _build.LIB_PATH


def load(build_if_missing: bool = True) -> C.CDLL:
    """Load liblspg.so (building it with nvcc first if the in-tree copy is absent or stale).

    There is deliberately no alternative implementation: if the library cannot be built or loaded the
    error propagates.
    """
    global _LIB
    if _LIB is not None:
        return _LIB
    path = library_path()
    if build_if_missing and _build.needs_build():
        try:
            _build.build_library()
        except Exception as exc:
            if not os.path.exists(path):
                raise
            # a stale library next to newer sources: usable (the GPU box has no reason to rebuild), but say so loudly
            import warnings
            warnings.warn(f"liblspg.so is older than its sources and could not be rebuilt ({exc}); using the existing binary",
                          RuntimeWarning)
    lib = C.CDLL(path)
    for name, argtypes in ARGTYPES.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = C.c_char_p if name.endswith("_last_error") else C.c_int
    _LIB = lib
    return lib


def check(code: int, prefix: str = "lspg") -> None:
    """Raise ``LspgError`` with ``<prefix>_last_error()`` if a ``<prefix>_*`` call returned ``code != 0``."""
    if code != 0:
        raise LspgError(code, (getattr(load(), prefix + "_last_error")() or b"").decode("utf-8", "replace"))


def cuda_device(device, what: str) -> torch.device:
    """``device`` (None: the current CUDA device) as an indexed CUDA device; anything else is refused, as there is no CPU
    path.  ``what`` names the caller in the refusal."""
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError(f"livespeechportraits_b200 has no CPU path: {what} needs an H100 (sm_90) device")
    return device if device.index is not None else torch.device("cuda", torch.cuda.current_device())


def to_device(x, device: torch.device, dtype=torch.float32) -> torch.Tensor:
    """``x`` (numpy, torch, any device) as a contiguous ``dtype`` tensor on ``device``.  A host array goes through pinned
    memory with a non-blocking copy, so the call does not wait for the device (a pageable copy would)."""
    t = torch.as_tensor(x)
    if t.device.type == "cpu":
        t = t.to(dtype=dtype).contiguous().pin_memory()
        return t.to(device=device, non_blocking=True)
    return t.to(device=device, dtype=dtype).contiguous()


def reserve(buf: Optional[torch.Tensor], nbytes: int, device: torch.device) -> torch.Tensor:
    """``buf`` if it holds at least ``nbytes`` bytes, else a new uint8 device buffer of ``nbytes`` (at least one byte).
    A stream keeps its workspaces this way: after its largest push nothing is allocated per push, so its device memory
    stays the same from push to push."""
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=device)
    return buf


def tensor_array(state_dict) -> Tuple[C.Array, list]:
    """A state dict as the ``lspg_tensor`` array of the ``*_load_weights`` calls: fp32 contiguous CPU copies, without
    BatchNorm's ``num_batches_tracked``.  The array points into ``keep``, which must outlive the call."""
    keep = [(k.encode(), v.detach().to(device="cpu", dtype=torch.float32).contiguous())
            for k, v in state_dict.items() if not k.endswith("num_batches_tracked")]
    arr = (LspgTensor * len(keep))()
    for e, (name, t) in zip(arr, keep):
        e.name, e.data, e.numel = name, C.cast(t.data_ptr(), C.POINTER(C.c_float)), t.numel()
    return arr, keep


def cached(cache: dict, net, make, extra=()):
    """The handle ``make(state_dict)`` built for the torch module ``net``, kept as the only entry of ``cache``.  It is
    re-loaded (``load_state_dict``) when the module's tensors changed - version counters move on every in-place write
    (load_state_dict, optimiser steps, init_weights), data pointers on re-allocation (``.to()``) - and rebuilt when
    ``extra`` changed."""
    sd = net.state_dict()
    stamp = (tuple((v.data_ptr(), v._version) for v in sd.values()), tuple(extra))
    hit = cache.get(id(net))
    if hit is None or hit[1] != stamp:
        if hit is not None and hit[1][1] == stamp[1]:
            gen = hit[0]
            gen.load_state_dict(sd)
        else:
            gen = make(sd)
        cache.clear()
        cache[id(net)] = (gen, stamp)
    return cache[id(net)][0]


class Handle:
    """Owns one native handle of the C ABI ``<prefix>_*``: ``__init__`` resolves the device (-1: a host-only handle,
    ``self.device`` None), ``_create`` calls ``<prefix>_create(&handle, *args, device)``, ``call`` makes checked calls
    with the handle first, ``cuda_stream`` enters the device and yields its current CUDA stream, and ``__del__``
    destroys it.  (``stream()`` on the subclasses opens an audio stream.)"""
    prefix = ""
    what = ""                      # names the subclass in the "no CPU path" refusal
    _handle = None

    def __init__(self, device):
        self._lib = load()
        self.device = None if device == -1 else cuda_device(device, self.what)

    def _create(self, *args) -> None:
        h = C.c_void_p()
        check(getattr(self._lib, self.prefix + "_create")(C.byref(h), *args, -1 if self.device is None else self.device.index),
              self.prefix)
        self._handle = h

    def call(self, name: str, *args) -> None:
        check(getattr(self._lib, f"{self.prefix}_{name}")(self._handle, *args), self.prefix)

    @contextlib.contextmanager
    def cuda_stream(self):
        """Enters the handle's device and yields its current stream (a ``cudaStream_t`` as int)."""
        with torch.cuda.device(self.device):
            yield torch.cuda.current_stream(self.device).cuda_stream

    def workspace_bytes(self, *args) -> int:
        """``<prefix>_workspace_bytes(handle, *args)``."""
        need = C.c_size_t()
        self.call("workspace_bytes", *args, C.byref(need))
        return need.value

    def workspace(self, *args) -> torch.Tensor:
        """A device buffer of the ``<prefix>_workspace_bytes(handle, *args)`` bytes (at least one byte)."""
        return torch.empty(max(self.workspace_bytes(*args), 1), dtype=torch.uint8, device=self.device)

    def __del__(self):
        try:
            if self._handle:
                getattr(self._lib, self.prefix + "_destroy")(self._handle)
                self._handle = None
        except Exception:
            pass
