"""Drop-in replacement for the reference's ``models/feature2face_G.py:Feature2Face_G``.

Same constructor (``Feature2Face_G(opt)``, reads ``opt.size / ngf / n_downsample_G / fp16 / isTrain``,
reference lines 8-21), same ``state_dict`` key grammar (``netG.model.model.<i>...``, so
``BaseModel.load_networks`` - models/base_model.py:193-223 - works unchanged, with or without the
DataParallel ``module.`` prefix), same ``forward(input[B,13,H,W] fp32) -> [B,3,H,W] fp32`` contract
(lines 27-34) and the same behaviour under ``networks.init_net`` (models/networks.py:382-402: ``.to(gpu)``,
optional ``DataParallel`` wrap, ``init_weights`` finds real ``Conv2d``/``BatchNorm2d`` leaves).

The module tree only HOLDS parameters.  ``forward`` never runs a torch op on them: it hands device pointers
to the C-ABI library (include/lspg.h), which runs the hand-written sm_90a kernels on the current CUDA stream.
There is no CPU or eager fallback: a CPU input, a device other than sm_90 (H100) or a missing library raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from . import _lib

KIND_HEAD, KIND_S1, KIND_S2, KIND_UP, KIND_TAIL = range(5)


class _Holder(nn.Module):
    """Anonymous container node of the parameter tree (stands where nn.Sequential / blocks stand upstream)."""

    def forward(self, *a, **k):  # pragma: no cover - never called
        raise RuntimeError("parameter holder; the generator runs through liblspg")


def _default_mode(opt) -> str:
    env = os.environ.get("LSP_B200_PRECISION")
    if env:
        if env not in _lib.LSPG_MODE:
            raise ValueError(f"LSP_B200_PRECISION must be one of {sorted(_lib.LSPG_MODE)}")
        return env
    # opt.fp16 (reference: torch.cuda.amp.autocast, feature2face_G.py:28-30) = caller accepts reduced precision
    return "fast" if getattr(opt, "fp16", 0) else "parity"


class Feature2Face_G(nn.Module):
    def __init__(self, opt, precision: Optional[str] = None):
        super().__init__()
        self.opt = opt
        self.isTrain = getattr(opt, "isTrain", False)
        size = getattr(opt, "size", "normal")
        if size not in _lib.LSPG_VARIANT:
            raise NotImplementedError(
                f"opt.size={size!r}: only 'normal' and 'large' are built for H100 (the 'small' U-Net takes a 23-channel "
                "input that no shipped config produces)")
        self.variant = size
        self.ngf = int(getattr(opt, "ngf", 64))
        self.num_downs = int(getattr(opt, "n_downsample_G", 8))
        self.in_nc, self.out_nc = 13, 3                      # feature2face_G.py:18-21
        self.precision = precision or _default_mode(opt)
        self._lib = _lib.load()
        self._handle = C.c_void_p()
        self._device_index: Optional[int] = None
        self._weights_dirty = True
        self._workspaces: Dict[Tuple[int, int, int, int, int], torch.Tensor] = {}
        self._host_handle = None
        # host-only handle: gives the layer list (keys, shapes) without needing a GPU
        plan = C.c_void_p()
        _lib.check(self._lib.lspg_create(C.byref(plan), _lib.LSPG_VARIANT[size], self.ngf, self.num_downs, self.in_nc,
                                         self.out_nc, -1))
        try:
            self._build_parameter_tree(plan)
        finally:
            self._lib.lspg_destroy(plan)

    # ------------------------------------------------------------------ parameter tree
    def _build_parameter_tree(self, plan) -> None:
        n = C.c_int()
        _lib.check(self._lib.lspg_num_layers(plan, C.byref(n)))
        info = _lib.LspgLayerInfo()
        for i in range(n.value):
            _lib.check(self._lib.lspg_layer_info_get(plan, i, C.byref(info)))
            cin = self.in_nc if info.kind == KIND_HEAD else info.cin[0] + (info.cin[1] if info.n_src == 2 else 0)
            stride = 2 if info.kind in (KIND_HEAD, KIND_S2) else 1
            self._attach(info.conv_key.decode(), nn.Conv2d(cin, info.cout, 3, stride, 1, bias=False))
            if info.has_bn:
                self._attach(info.bn_key.decode(), nn.BatchNorm2d(info.cout))

    def _attach(self, dotted: str, leaf: nn.Module) -> None:
        node: nn.Module = self
        parts = dotted.split(".")
        for p in parts[:-1]:
            if p not in node._modules:
                node.add_module(p, _Holder())
            node = node._modules[p]
        node.add_module(parts[-1], leaf)

    # ------------------------------------------------------------------ weight tracking
    def mark_weights_dirty(self) -> None:
        """Call after editing parameters in place; load_state_dict/.to()/.eval() do it automatically."""
        self._weights_dirty = True

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        out = super().load_state_dict(state_dict, strict=strict, **kw)
        self._weights_dirty = True
        return out

    def _load_from_state_dict(self, *a, **k):
        # reached for every module of the tree when ANY ancestor's load_state_dict runs (e.g. the
        # nn.DataParallel wrapper networks.init_net creates, whose load never calls the override above)
        self._weights_dirty = True
        return super()._load_from_state_dict(*a, **k)

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        self._weights_dirty = True
        return out

    def train(self, mode: bool = True):
        self._weights_dirty = True
        return super().train(mode)

    # ------------------------------------------------------------------ copies, replicas, pickling
    # The native handle (packed weights, plans, CUDA graphs) and the workspaces belong to ONE module object.  A shallow
    # copy that shared them would double-free the handle; so every way of copying the module resets the native state and
    # the copy re-creates its own handle on first use.
    _NATIVE_STATE = ("_lib", "_handle", "_host_handle", "_workspaces", "_device_index", "_weights_dirty")

    def __getstate__(self):
        d = self.__dict__.copy()
        for k in self._NATIVE_STATE:
            d.pop(k, None)
        return d

    def __setstate__(self, state):
        super().__setstate__(state)
        self._lib = _lib.load()
        self._handle = C.c_void_p()
        self._host_handle = None
        self._device_index = None
        self._weights_dirty = True
        self._workspaces = {}

    def __deepcopy__(self, memo):
        import copy
        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        new.__setstate__(copy.deepcopy(self.__getstate__(), memo))
        return new

    def _replicate_for_data_parallel(self):
        # nn.DataParallel with more than one device id shallow-copies __dict__ (shared native handle) and strips the
        # parameters from the replicas (they would upload empty weights).  The reference's multi-GPU hook
        # (models/networks.py:392-401) is replaced by one process per GPU: parallel.ShardedRenderer.
        raise NotImplementedError(
            "Feature2Face_G (H100) cannot be replicated by nn.DataParallel over several devices: the module owns a native "
            "handle per device.  Wrap it with device_ids=[one id] (what demo.py does) or shard frames over processes with "
            "livespeechportraits_b200.parallel.ShardedRenderer")

    def _ensure_handle(self, device: torch.device) -> None:
        idx = _lib.cuda_device(device, "the generator's input").index
        if self._handle and self._device_index == idx:
            return
        if self._handle:
            self._drop_workspaces()
            self._lib.lspg_destroy(self._handle)
            self._handle = C.c_void_p()
        h = C.c_void_p()
        _lib.check(self._lib.lspg_create(C.byref(h), _lib.LSPG_VARIANT[self.variant], self.ngf, self.num_downs, self.in_nc,
                                         self.out_nc, idx))
        self._handle, self._device_index = h, idx
        self._weights_dirty = True
        self._workspaces.clear()

    def _push_weights(self) -> None:
        arr, _keep = _lib.tensor_array(super().state_dict())
        _lib.check(self._lib.lspg_load_weights(self._handle, arr, len(arr)))
        self._weights_dirty = False

    # ------------------------------------------------------------------ forward
    MAX_WORKSPACES = 4

    def _drop_workspaces(self) -> None:
        if self._handle and self._workspaces:
            _lib.check(self._lib.lspg_release_workspace(self._handle, None))     # waits for the device, drops every plan
        self._workspaces.clear()

    def _workspace(self, batch: int, height: int, width: int, mode: int) -> torch.Tensor:
        """Caller-owned scratch of one problem size, LRU-cached.  Before a workspace is released the library is told
        (lspg_release_workspace: device sync + the plans / graphs that point into it are dropped), so no kernel that is
        still in flight on another stream can see its memory reused."""
        key = (batch, height, width, mode, self._device_index)
        ws = self._workspaces.pop(key, None)
        if ws is None:
            need = C.c_size_t()
            _lib.check(self._lib.lspg_workspace_bytes(self._handle, batch, height, width, mode, C.byref(need)))
            while len(self._workspaces) >= self.MAX_WORKSPACES:
                old_key = next(iter(self._workspaces))               # least recently used (dict keeps insertion order)
                old = self._workspaces.pop(old_key)
                _lib.check(self._lib.lspg_release_workspace(self._handle, old.data_ptr()))
                del old
            ws = torch.empty(need.value, dtype=torch.uint8, device=torch.device("cuda", self._device_index))
        self._workspaces[key] = ws                                   # (re)insert as most recently used
        return ws

    def render_image(self, feature_map: torch.Tensor, cand_image: Optional[torch.Tensor], out: Optional[torch.Tensor] = None,
                     precision: Optional[str] = None) -> torch.Tensor:
        """``render`` + ``util.tensor2im`` (util/util.py:19-42) fused into the last kernel: uint8 ``[B,H,W,3]`` images
        (``(x+1)/2*255``, clip, truncate, HWC) instead of fp32 ``[B,3,H,W]`` - what demo.py:268 builds per frame."""
        return self.render(feature_map, cand_image, out=out, precision=precision, _uint8=True)

    def render_into_ptr(self, feature_map: torch.Tensor, cand_image: Optional[torch.Tensor], out_ptr: int,
                        precision: Optional[str] = None) -> None:
        """``render`` with the fp32 ``[B,3,H,W]`` output written through a raw device address (8-byte aligned) instead of a
        tensor: the address may be an NVLink *multicast* mapping (``torch.distributed._symmetric_memory`` handle
        ``.multicast_ptr`` + offset), in which case every float2 store of the tail kernel's epilogue lands in the clip buffer
        of EVERY rank - the all-gather happens inside the conv kernel (parallel.ShardedRenderer, gather="mc")."""
        if int(out_ptr) % 8:
            raise ValueError("out_ptr must be 8-byte aligned")
        self.render(feature_map, cand_image, precision=precision, _out_ptr=int(out_ptr))

    def render(self, feature_map: torch.Tensor, cand_image: Optional[torch.Tensor], out: Optional[torch.Tensor] = None,
               precision: Optional[str] = None, _uint8: bool = False, _out_ptr: Optional[int] = None) -> torch.Tensor:
        """Fused ``torch.cat([feature_map, cand_image], 1)`` + generator (feature2face_model.py:231-233).

        ``cand_image`` may have batch 1 (broadcast over the frames, as demo.py:266 reuses one candidate set).
        """
        if self.training:
            raise NotImplementedError("training-mode BatchNorm is not implemented: call .eval() (inference path only)")
        if feature_map.dtype != torch.float32 or (cand_image is not None and cand_image.dtype != torch.float32):
            raise TypeError("inputs must be fp32 (reference contract)")
        self._ensure_handle(feature_map.device)
        if self._weights_dirty:
            self._push_weights()
        if cand_image is None:
            if feature_map.dim() != 4 or feature_map.shape[1] != self.in_nc:
                raise ValueError(f"expected [B,{self.in_nc},H,W] input, got {tuple(feature_map.shape)}")
            x = self._aligned(feature_map.contiguous())
            b, _, h, w = x.shape
            fm_ptr, fm_stride = x.data_ptr(), self.in_nc * h * w
            cand_ptr, cand_stride = x.data_ptr() + 4 * h * w, self.in_nc * h * w
            hold = (x,)
        else:
            fm = self._aligned(feature_map.contiguous())
            cd = self._aligned(cand_image.contiguous())
            b, c1, h, w = fm.shape
            if c1 != 1 or cd.shape[1] != self.in_nc - 1 or cd.shape[2:] != fm.shape[2:] or cd.shape[0] not in (1, b):
                raise ValueError(f"expected [B,1,H,W] + [B|1,{self.in_nc - 1},H,W], got {tuple(fm.shape)} + {tuple(cd.shape)}")
            if cd.device != fm.device:
                raise ValueError("feature_map and cand_image must be on the same device")
            fm_ptr, fm_stride = fm.data_ptr(), h * w
            cand_ptr, cand_stride = cd.data_ptr(), (0 if cd.shape[0] == 1 and b > 1 else (self.in_nc - 1) * h * w)
            hold = (fm, cd)
        mode = _lib.LSPG_MODE[precision or self.precision]
        ws = self._workspace(b, h, w, mode)
        oshape, odtype = ((b, h, w, self.out_nc), torch.uint8) if _uint8 else ((b, self.out_nc, h, w), torch.float32)
        user_out = None
        if _out_ptr is not None:
            if _uint8 or out is not None:
                raise ValueError("raw output address: fp32 frames only, no `out` tensor")
            stream = torch.cuda.current_stream(feature_map.device).cuda_stream
            _lib.check(self._lib.lspg_forward(self._handle, fm_ptr, fm_stride, cand_ptr, cand_stride, _out_ptr, b, h, w,
                                              ws.data_ptr(), ws.numel(), mode, stream))
            del hold
            return None
        if out is None:
            out = torch.empty(oshape, dtype=odtype, device=feature_map.device)
        elif tuple(out.shape) != oshape or out.dtype != odtype or not out.is_contiguous():
            raise ValueError(f"out must be a contiguous {odtype} tensor of shape {oshape}")
        elif out.device != feature_map.device:
            raise ValueError(f"out is on {out.device}, the inputs are on {feature_map.device}: the kernels write `out` through a raw pointer")
        elif out.data_ptr() % 8:
            # the tail kernel stores float2 / 2-byte pairs: a view at an odd storage offset goes through a temporary
            user_out, out = out, torch.empty(oshape, dtype=odtype, device=feature_map.device)
        stream = torch.cuda.current_stream(feature_map.device).cuda_stream
        fn = self._lib.lspg_forward_image if _uint8 else self._lib.lspg_forward
        _lib.check(fn(self._handle, fm_ptr, fm_stride, cand_ptr, cand_stride, out.data_ptr(), b, h, w,
                      ws.data_ptr(), ws.numel(), mode, stream))
        del hold
        if user_out is not None:
            user_out.copy_(out)
            return user_out
        return out

    @staticmethod
    def _aligned(t: torch.Tensor) -> torch.Tensor:
        """The input packer reads float2: a contiguous view that starts at an odd element of its storage is copied."""
        return t if t.data_ptr() % 8 == 0 else t.clone()

    def graph_stats(self) -> dict:
        """CUDA-graph bookkeeping of the native handle: captures, in-place I/O pointer updates, forced re-captures."""
        a, b_, c = C.c_int64(), C.c_int64(), C.c_int64()
        _lib.check(self._lib.lspg_graph_stats(self._handle, C.byref(a), C.byref(b_), C.byref(c)))
        return {"captures": a.value, "io_updates": b_.value, "recaptures": c.value}

    def draw_feature_maps(self, landmarks: torch.Tensor, shoulders: Optional[torch.Tensor] = None,
                          size: tuple = (512, 512), out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Rasterise a clip's landmark tracks into the ``[B,1,H,W]`` {0,1} maps ``render`` consumes, on the GPU.

        Batched replacement of ``FaceDataset.get_data_test_mode`` (datasets/face_dataset.py:276-323; 88 ``cv2.line`` calls and
        a 1 MB host->device copy per frame at demo.py:262-265), bit-exact with cv2.  ``landmarks`` ``[B,73,2]`` and
        ``shoulders`` ``[B,2k,2]`` (or None) are fp32 CUDA tensors in pixel coordinates; ``size`` is ``(W, H)`` like the
        reference's ``(opt.loadSize, opt.loadSize)``."""
        if landmarks.dtype != torch.float32 or landmarks.dim() != 3 or landmarks.shape[1:] != (73, 2):
            raise ValueError(f"landmarks must be fp32 [B,73,2], got {landmarks.dtype} {tuple(landmarks.shape)}")
        self._ensure_handle(landmarks.device)
        b = landmarks.shape[0]
        w, h = int(size[0]), int(size[1])
        lm = landmarks.contiguous()
        sh, n_sh = None, 0
        if shoulders is not None:
            if shoulders.dtype != torch.float32 or shoulders.dim() != 3 or shoulders.shape[0] != b or shoulders.shape[2] != 2 \
                    or shoulders.shape[1] % 2 or shoulders.device != landmarks.device:
                raise ValueError(f"shoulders must be fp32 [B,2k,2] on the landmarks' device, got {tuple(shoulders.shape)}")
            sh, n_sh = shoulders.contiguous(), shoulders.shape[1]
        if out is None:
            out = torch.empty((b, 1, h, w), dtype=torch.float32, device=landmarks.device)
        elif tuple(out.shape) != (b, 1, h, w) or out.dtype != torch.float32 or not out.is_contiguous() \
                or out.device != landmarks.device:
            raise ValueError(f"out must be a contiguous fp32 tensor of shape {(b, 1, h, w)} on {landmarks.device}")
        stream = torch.cuda.current_stream(landmarks.device).cuda_stream
        _lib.check(self._lib.lspg_draw_feature_maps(self._handle, lm.data_ptr(), sh.data_ptr() if sh is not None else None, n_sh,
                                                    out.data_ptr(), b, h, w, stream))
        del lm, sh
        return out

    def forward(self, input: torch.Tensor) -> torch.Tensor:  # noqa: A002 - reference argument name
        return self.render(input, None)

    # ------------------------------------------------------------------ introspection used by tests / bench
    def _info_handle(self):
        """Device handle if one exists, else a host-only handle (structure queries need no GPU)."""
        if self._handle:
            return self._handle
        if not getattr(self, "_host_handle", None):
            h = C.c_void_p()
            _lib.check(self._lib.lspg_create(C.byref(h), _lib.LSPG_VARIANT[self.variant], self.ngf, self.num_downs,
                                             self.in_nc, self.out_nc, -1))
            self._host_handle = h
        return self._host_handle

    def launches_per_forward(self) -> int:
        n = C.c_int()
        _lib.check(self._lib.lspg_launches_per_forward(self._info_handle(), C.byref(n)))
        return n.value

    def flops_per_frame(self, height: int, width: int) -> float:
        v = C.c_double()
        _lib.check(self._lib.lspg_flops_per_frame(self._info_handle(), height, width, C.byref(v)))
        return v.value

    def profile_enable(self, enabled: bool = True) -> None:
        """Record CUDA events around every kernel of subsequent forwards (lspg_profile_enable)."""
        _lib.check(self._lib.lspg_profile_enable(self._handle, 1 if enabled else 0))

    def profile_read(self) -> Tuple[List[float], int]:
        """(average ms per launch [input packer, conv 0, conv 1, ...], forwards averaged); resets the record."""
        nl = C.c_int()
        _lib.check(self._lib.lspg_num_layers(self._info_handle(), C.byref(nl)))
        n = nl.value + 1                         # input packer + one slot per conv layer (incl. its split-K finisher)
        buf = (C.c_float * n)()
        cnt = C.c_int()
        _lib.check(self._lib.lspg_profile_read(self._handle, buf, n, C.byref(cnt)))
        return list(buf), cnt.value

    def layer_table(self, height: int, width: int) -> List[dict]:
        """One dict per conv launch: kind, state-dict key, channels, output grid and algorithmic FLOPs per frame."""
        hdl = self._info_handle()
        n = C.c_int()
        _lib.check(self._lib.lspg_num_layers(hdl, C.byref(n)))
        rows = []
        info = _lib.LspgLayerInfo()
        for i in range(n.value):
            _lib.check(self._lib.lspg_layer_info_get(hdl, i, C.byref(info)))
            cin = self.in_nc if info.kind == KIND_HEAD else info.cin[0] + (info.cin[1] if info.n_src == 2 else 0)
            if info.out >= 0:
                c, th, tw = C.c_int(), C.c_int(), C.c_int()
                _lib.check(self._lib.lspg_tensor_shape(hdl, info.out, height, width, C.byref(c), C.byref(th), C.byref(tw)))
                oh, ow = th.value, tw.value
            else:
                oh, ow = height, width
            rows.append(dict(kind=info.kind, key=info.conv_key.decode(), cin=cin, cout=info.cout, out_h=oh, out_w=ow,
                             flops=2.0 * oh * ow * info.cout * cin * 9, src=[info.src[0], info.src[1]][: info.n_src],
                             out=info.out, res=info.res))
        return rows

    def debug_read_tensor(self, tensor_id: int, batch: int, height: int, width: int, limb: int = 0,
                          precision: Optional[str] = None) -> torch.Tensor:
        """Activation tensor of the most recent forward: fp16 limbs after a PARITY forward, bf16 after a FAST one."""
        c, th, tw = C.c_int(), C.c_int(), C.c_int()
        _lib.check(self._lib.lspg_tensor_shape(self._handle, tensor_id, height, width, C.byref(c), C.byref(th), C.byref(tw)))
        dt = torch.float16 if (precision or self.precision) == "parity" else torch.bfloat16
        buf = torch.empty((batch, th.value, tw.value, c.value), dtype=dt)
        _lib.check(self._lib.lspg_debug_read_tensor(self._handle, tensor_id, limb, buf.data_ptr(), buf.numel()))
        return buf

    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                self._lib.lspg_destroy(self._handle)
                self._handle = C.c_void_p()
            if getattr(self, "_host_handle", None):
                self._lib.lspg_destroy(self._host_handle)
        except Exception:
            pass


def install(models_module_name: str = "models.feature2face_G") -> None:
    """Swap the reference's generator class for this one; ``demo.py`` then runs unchanged.

    ``models/feature2face_model.py:27`` resolves ``feature2face_G.Feature2Face_G`` at call time, so replacing the
    module attribute before ``create_model(opt)`` is enough.
    """
    import importlib

    mod = importlib.import_module(models_module_name)
    mod.Feature2Face_G = Feature2Face_G
