"""The recurrent audio networks on the GPU (demo.py stages 1 and 3): the APC encoder's GRU stack
(``APC_encoder``, models/networks.py:20-69) and Audio2Mouth (``Audio2Feature`` with the LSTM decoder,
models/audio2feature.py:32-69, as ``Audio2FeatureModel.generate_sequences`` drives it, models/audio2feature_model.py:117-154).

Each recurrent layer is one input-projection GEMM over the whole clip plus one persistent thread-block cluster kernel that
runs every time step (include/lspr.h, csrc/lspr.cu); the MLPs around the LSTM are GEMMs with eval-mode BatchNorm folded
into their epilogue.  ``ApcEncoder.forward`` and ``MouthGenerator.generate`` take and return CUDA tensors and make no
host-synchronising call, so wav -> mel -> APC -> manifold projection -> mouth track stays on the device.

``install()`` swaps ``APC_encoder.forward`` and ``Audio2FeatureModel.generate_sequences`` for drop-ins with the reference's
signatures and return types; the weights come from the (unmodified) modules, re-packed whenever they change.  There is no
CPU path.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict

import numpy as np
import torch

from . import _lib

LSTM_HIDDEN = 256          # models/audio2feature.py:40


def _cuda_device(device) -> torch.device:
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("livespeechportraits_b200 has no CPU path: the recurrent networks need an H100 (sm_90) device")
    return device if device.index is not None else torch.device("cuda", torch.cuda.current_device())


class _Recurrent:
    """Owns one native handle (packed weights on one device)."""

    def __init__(self, cfg: _lib.LsprConfig, state_dict: Dict[str, torch.Tensor], device):
        self._lib = _lib.load()
        self._handle = C.c_void_p()
        self.cfg = cfg
        self.device = _cuda_device(device) if device != -1 else None
        _lib.check_r(self._lib.lspr_create(C.byref(self._handle), C.byref(cfg), self.device.index if self.device else -1))
        self.load_state_dict(state_dict)

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor]) -> None:
        names, keep = [], []
        for k, v in state_dict.items():
            if k.endswith("num_batches_tracked"):
                continue
            names.append(k.encode())
            keep.append(v.detach().to(device="cpu", dtype=torch.float32).contiguous())
        arr = (_lib.LspgTensor * len(keep))()
        for i, (nm, t) in enumerate(zip(names, keep)):
            arr[i].name = nm
            arr[i].data = C.cast(t.data_ptr(), C.POINTER(C.c_float))
            arr[i].numel = t.numel()
        _lib.check_r(self._lib.lspr_load_weights(self._handle, arr, len(keep)))

    def packed(self, which: int) -> np.ndarray:
        """The array ``lspr_debug_packed`` returns (see include/lspr.h for the order)."""
        n = C.c_int64()
        _lib.check_r(self._lib.lspr_debug_packed(self._handle, which, None, C.byref(n)))
        out = np.empty(n.value, np.float32)
        _lib.check_r(self._lib.lspr_debug_packed(self._handle, which, out.ctypes.data, C.byref(n)))
        return out

    def _run(self, x: torch.Tensor, width: int, out_shape, cluster: int) -> torch.Tensor:
        if not isinstance(x, torch.Tensor) or not x.is_cuda:
            raise RuntimeError("input must be a CUDA tensor (there is no CPU path)")
        if self.device is None:
            raise RuntimeError("host-only handle: created with device=-1")
        if x.dim() != 2 or x.shape[1] != width:
            raise ValueError(f"input must be [n, {width}], got {tuple(x.shape)}")
        x = x.to(device=self.device, dtype=torch.float32).contiguous()
        if x.data_ptr() % 16:
            x = x.clone()
        n = x.shape[0]
        out = torch.empty(out_shape, dtype=torch.float32, device=self.device)
        nbytes = C.c_size_t()
        _lib.check_r(self._lib.lspr_workspace_bytes(self._handle, n, C.byref(nbytes)))
        ws = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device).cuda_stream
            _lib.check_r(self._lib.lspr_forward(self._handle, x.data_ptr(), n, out.data_ptr(), ws.data_ptr(), nbytes.value,
                                                int(cluster), stream))
        self._keep = (x, ws)           # inputs stay alive until the caller synchronises on the result
        return out

    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                self._lib.lspr_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass


class ApcEncoder(_Recurrent):
    """``APC_encoder`` on one clip.  ``state_dict`` uses its key grammar (``rnns.{i}.weight_ih_l0``, ...; an optional
    ``module.`` prefix is accepted); the layer count and mel width are read from it.  ``device=-1`` makes a host-only
    handle (packing introspection)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device=None, residual: bool = False):
        sd = {k[7:] if k.startswith("module.") else k: v for k, v in state_dict.items()}
        layers = 0
        while f"rnns.{layers}.weight_ih_l0" in sd:
            layers += 1
        if layers == 0:
            raise ValueError("state_dict has no rnns.0.weight_ih_l0")
        cfg = _lib.LsprConfig()
        cfg.kind = _lib.LSPR_KIND["apc"]
        cfg.input_dim = int(sd["rnns.0.weight_ih_l0"].shape[1])
        cfg.hidden = int(sd["rnns.0.weight_hh_l0"].shape[1])
        cfg.num_layers = layers
        cfg.residual = 1 if residual else 0
        self.mel_dim, self.hidden = cfg.input_dim, cfg.hidden
        super().__init__(cfg, state_dict, device)

    def forward(self, mel: torch.Tensor, cluster: int = 0) -> torch.Tensor:
        """mel [T, mel_dim] CUDA -> features [T, hidden] CUDA fp32, enqueued on the current stream.  ``cluster``: CTAs
        per recurrence launch (0 = library choice, 8 or 16)."""
        return self._run(mel, self.mel_dim, (mel.shape[0], self.hidden), cluster)

    __call__ = forward


def mouth_output_size(opt) -> int:
    """models/audio2feature.py:11-15."""
    if getattr(opt, "loss", "L2") == "GMM":
        return (2 * int(opt.A2L_GMM_ndim) + 1) * int(opt.A2L_GMM_ncenter)
    return int(opt.A2L_GMM_ndim) * int(getattr(opt, "predict_length", 1))


class MouthGenerator(_Recurrent):
    """Audio2Mouth: ``Audio2Feature`` with ``feature_decoder='LSTM'`` as ``generate_sequences`` runs it.  ``state_dict``
    uses its key grammar (``downsample.0.weight``, ``LSTM.weight_ih_l0``, ``fc.1.running_var``, ...)."""

    def __init__(self, opt, state_dict: Dict[str, torch.Tensor], device=None):
        if getattr(opt, "feature_decoder", "LSTM") != "LSTM":
            raise NotImplementedError("Audio2Mouth runs on H100 with the LSTM decoder (the shipped default) only")
        cfg = _lib.LsprConfig()
        cfg.kind = _lib.LSPR_KIND["mouth"]
        cfg.input_dim = int(getattr(opt, "APC_hidden_size", 512))
        cfg.frame_future = int(getattr(opt, "frame_future", 18))
        cfg.out_dim = mouth_output_size(opt)
        self.apc_hidden, self.frame_future, self.out_dim = cfg.input_dim, cfg.frame_future, cfg.out_dim
        super().__init__(cfg, state_dict, device)

    def generate(self, feats: torch.Tensor) -> torch.Tensor:
        """APC features [n, APC_hidden] CUDA (n even) -> predictions [n / 2, out] CUDA fp32: the rows
        ``generate_sequences`` returns, enqueued on the current stream."""
        n = int(feats.shape[0])
        if n % 2:
            total = (n + 2 * self.frame_future) * self.apc_hidden           # what models/audio2feature.py:65 raises
            raise RuntimeError(f"shape '[1, -1, {2 * self.apc_hidden}]' is invalid for input of size {total}")
        if n < 2:
            raise ValueError("need at least 2 APC rows")
        return self._run(feats, self.apc_hidden, (n // 2, self.out_dim), 0)


# ------------------------------------------------------------------------------------------------------------------
# Drop-ins for the reference modules
# ------------------------------------------------------------------------------------------------------------------
_APC: "Dict[int, tuple]" = {}          # id(module) -> (ApcEncoder, stamp)
_MOUTH: "Dict[int, tuple]" = {}        # id(module) -> (MouthGenerator, stamp)


def _cached(cache: dict, net, make, extra=()):
    """The handle for ``net``, re-packed when its tensors changed: version counters move on every in-place write
    (load_state_dict, optimiser steps), data pointers on re-allocation (``.to()``)."""
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


def apc_forward(self, inputs, lengths):
    """Replacement for ``APC_encoder.forward`` (models/networks.py:37-69), bound by ``install()``: inputs
    [1, T, mel_dim] on a CUDA device, lengths [T] -> [1, T, hidden] fp32 on the input's device."""
    if not isinstance(inputs, torch.Tensor) or not inputs.is_cuda:
        raise RuntimeError("H100 APC encoder: the input must be a CUDA tensor (there is no CPU path)")
    if inputs.dim() != 3 or inputs.shape[0] != 1:
        raise ValueError(f"H100 APC encoder: batch 1 only, got input shape {tuple(inputs.shape)}")
    lens = torch.as_tensor(lengths).reshape(-1)
    if lens.numel() != 1 or int(lens[0]) != inputs.shape[1]:
        raise ValueError(f"H100 APC encoder: lengths must be [{inputs.shape[1]}] (the full clip), got {lens.tolist()}")
    enc = _cached(_APC, self, lambda sd: ApcEncoder(sd, inputs.device, residual=bool(self.rnn_residual)),
                  (bool(self.rnn_residual), str(inputs.device)))
    return enc.forward(inputs[0])[None]


def generate_sequences(self, audio_feats, sample_rate=16000, fps=60, fill_zero=True, opt=[]):   # noqa: B006 - reference signature
    """Replacement for ``Audio2FeatureModel.generate_sequences`` (models/audio2feature_model.py:117-154), bound by
    ``install()``.  Same arguments, same return value ([nframe, output_size] float32 numpy)."""
    net = self.Audio2Feature.module if hasattr(self.Audio2Feature, "module") else self.Audio2Feature
    mopt = getattr(net, "opt", opt)
    if getattr(mopt, "feature_decoder", "LSTM") != "LSTM":
        raise NotImplementedError("H100 Audio2Mouth: LSTM decoder only (WaveNet is not built)")
    device = torch.device(getattr(self, "device", "cuda"))
    if device.type != "cuda":
        raise RuntimeError("H100 Audio2Mouth: the model is on the CPU (there is no CPU path)")
    net.eval()                                                                          # :139
    ff = int(opt.frame_future)

    def make(sd):
        o = _OptView(mopt, frame_future=ff)
        return MouthGenerator(o, sd, device)
    gen = _cached(_MOUTH, net, make, (ff, str(device)))
    feats = torch.as_tensor(np.asarray(audio_feats)).to(device=device, dtype=torch.float32)
    return gen.generate(feats).cpu().numpy()                                            # :147-149


class _OptView:
    """``opt`` with some fields replaced."""

    def __init__(self, base, **over):
        self._base, self._over = base, over

    def __getattr__(self, name):
        if name in self._over:
            return self._over[name]
        return getattr(self._base, name)


def install(networks_module: str = "models.networks", a2f_module: str = "models.audio2feature_model") -> None:
    """Swap the reference's APC encoder forward and Audio2Mouth generation for the CUDA ones; ``demo.py`` and
    ``predict.py`` then run unchanged."""
    import importlib
    importlib.import_module(networks_module).APC_encoder.forward = apc_forward
    importlib.import_module(a2f_module).Audio2FeatureModel.generate_sequences = generate_sequences
