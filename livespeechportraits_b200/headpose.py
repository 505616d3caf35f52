"""Audio2Headpose generation on the GPU (SURVEY.md 8f, row N4): drop-in for
``Audio2HeadposeModel.generate_sequences`` (models/audio2headpose_model.py:133-187).

The reference runs, per generated frame, a 255-step WaveNet forward, a ``.cpu()`` copy, ``Sample_GMM`` on the host and a
``torch.cat`` of the history - 672 iterations for the shipped clip.  ``generate_sequences`` below hands the whole clip to
ONE persistent CUDA kernel (include/lsph.h, csrc/lsph.cu) and keeps the reference's signature, return type
(``[nframe, ndim]`` float64 numpy) and random stream: the draws ``Sample_GMM`` would take from torch's global CPU generator
(``torch.multinomial`` then ``torch.randn`` per frame, models/losses.py:87,96) are taken here in the same order and passed
to the kernel, so a caller that seeds torch gets the sequence the reference's arithmetic would produce (up to fp32
summation order).  With more than one mixture component the component is chosen on the device from a U(0,1) draw per
frame (same distribution, not ``torch.multinomial``'s own stream).

``install()`` swaps the method on the reference's model class, the weights come from the model's own (unmodified)
``Audio2Headpose`` module - ``demo.py`` then runs unchanged.  There is no CPU path.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib


def config_from_opt(opt) -> _lib.LsphConfig:
    """The option fields Audio2Headpose.__init__ reads (models/audio2headpose.py:8-37)."""
    if getattr(opt, "feature_decoder", "WaveNet") != "WaveNet":
        raise NotImplementedError("only the WaveNet decoder (the shipped default) is built for H100; the LSTM decoder is not autoregressive")
    g = lambda k, d: int(getattr(opt, k, d))      # noqa: E731
    cfg = _lib.LsphConfig()
    cfg.apc_hidden = g("APC_hidden_size", 512)
    cfg.frame_future = g("frame_future", 15)
    cfg.layers = g("A2H_wavenet_residual_layers", 7)
    cfg.blocks = g("A2H_wavenet_residual_blocks", 2)
    cfg.residual_ch = g("A2H_wavenet_residual_channels", 128)
    cfg.dilation_ch = g("A2H_wavenet_dilation_channels", 128)
    cfg.skip_ch = g("A2H_wavenet_skip_channels", 256)
    cfg.kernel_size = g("A2H_wavenet_kernel_size", 2)
    cfg.use_bias = 1 if getattr(opt, "A2H_wavenet_use_bias", True) else 0
    cfg.cond_ch = g("A2H_wavenet_cond_channels", 512)
    cfg.input_ch = g("A2H_wavenet_input_channels", 12)
    cfg.ncenter = g("A2H_GMM_ncenter", 1)
    cfg.ndim = g("A2H_GMM_ndim", 12)
    cfg.loss_gmm = 1 if getattr(opt, "loss", "GMM") == "GMM" else 0
    return cfg


class HeadposeGenerator:
    """Owns the native handle (packed weights on one device).  ``state_dict`` uses the key grammar of
    ``Audio2Headpose(opt).state_dict()`` (an optional ``module.`` prefix is accepted)."""

    def __init__(self, opt, state_dict: Dict[str, torch.Tensor], device: Optional[torch.device] = None):
        self._lib = _lib.load()
        self._handle = C.c_void_p()
        self.cfg = config_from_opt(opt)
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("livespeechportraits_b200 has no CPU path: the headpose loop needs an H100 (sm_90) device")
        self.device = device if device.index is not None else torch.device("cuda", torch.cuda.current_device())
        _lib.check_h(self._lib.lsph_create(C.byref(self._handle), C.byref(self.cfg), self.device.index))
        rf = C.c_int()
        _lib.check_h(self._lib.lsph_receptive_field(self._handle, C.byref(rf)))
        self.receptive_field = rf.value
        self.out_channels = (2 * self.cfg.ndim + 1) * self.cfg.ncenter if self.cfg.loss_gmm else self.cfg.ndim
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
        _lib.check_h(self._lib.lsph_load_weights(self._handle, arr, len(keep)))

    def generate(self, audio_feats, pre_headpose, noise, sigma_scale: float, uniform=None, return_params: bool = False,
                 cluster: int = 0):
        """Device-level call: fp32 tensors (moved to the handle's device if needed).  ``audio_feats`` [n_audio, 2*APC_hidden],
        ``pre_headpose`` [input_ch], ``noise`` [nframe, ndim]; returns ``pred`` [nframe, ndim] (and the per-frame network
        output [nframe, out_ch]) as CUDA tensors, enqueued on the current stream."""
        dev = self.device
        to = lambda a: torch.as_tensor(a, dtype=torch.float32).to(dev).contiguous()      # noqa: E731
        a = to(audio_feats).reshape(-1, 2 * self.cfg.apc_hidden)
        n_audio = a.shape[0]
        nframe = n_audio - self.cfg.frame_future
        if nframe < 1:
            raise ValueError(f"need more than frame_future={self.cfg.frame_future} audio rows, got {n_audio}")
        pre = to(pre_headpose).reshape(-1)
        if pre.numel() != self.cfg.input_ch:
            raise ValueError(f"pre_headpose must have {self.cfg.input_ch} values")
        nz = to(noise).reshape(nframe, self.cfg.ndim) if noise is not None else torch.zeros((nframe, self.cfg.ndim), device=dev)
        un = to(uniform).reshape(nframe) if uniform is not None else None
        pred = torch.empty((nframe, self.cfg.ndim), dtype=torch.float32, device=dev)
        params = torch.empty((nframe, self.out_channels), dtype=torch.float32, device=dev) if return_params else None
        for t in (a, pre, nz):
            if t.data_ptr() % 16:
                raise ValueError("device buffers must be 16-byte aligned")
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check_h(self._lib.lsph_generate(self._handle, a.data_ptr(), n_audio, pre.data_ptr(), nz.data_ptr(),
                                                 un.data_ptr() if un is not None else None, float(sigma_scale), pred.data_ptr(),
                                                 params.data_ptr() if params is not None else None, int(cluster), stream))
        self._keep = (a, pre, nz, un)            # inputs stay alive until the caller synchronises on the result
        return (pred, params) if return_params else pred

    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                self._lib.lsph_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass


def draw_reference_noise(nframe: int, ndim: int, ncenter: int):
    """The draws Sample_GMM takes from torch's global CPU generator for ``nframe`` frames, in its order
    (models/losses.py:87 ``torch.multinomial`` then :96 ``torch.randn`` per frame).  Returns (noise [nframe, ndim],
    uniform [nframe] or None)."""
    noise = torch.empty((nframe, ndim), dtype=torch.float32)
    prob = torch.full((1, ncenter), 1.0 / ncenter)
    for i in range(nframe):
        torch.multinomial(prob, num_samples=1, replacement=True)
        noise[i] = torch.randn(1, ndim).float()[0]
    uniform = torch.rand(nframe) if ncenter > 1 else None
    return noise, uniform


_GENERATORS: "Dict[int, tuple]" = {}          # id(module) -> (HeadposeGenerator, stamp of the module's tensors)


def generate_sequences(self, audio_feats, pre_headpose, fill_zero=True, sigma_scale=0.0, opt=[]):   # noqa: B006 - reference signature
    """Replacement for ``Audio2HeadposeModel.generate_sequences`` (models/audio2headpose_model.py:133-187), bound to the
    reference model by ``install()``.  Same arguments, same return value ([nframe, A2H_GMM_ndim] float64 numpy)."""
    if getattr(opt, "feature_decoder", "WaveNet") != "WaveNet":
        raise NotImplementedError("H100 headpose loop: WaveNet decoder only")
    if not fill_zero:
        return None                                                                    # audio2headpose_model.py:161-162
    net = self.Audio2Headpose.module if hasattr(self.Audio2Headpose, "module") else self.Audio2Headpose
    sd = net.state_dict()
    # the packed copy on the device is reused while the module's tensors are untouched: tensor version counters move on every
    # in-place write (load_state_dict copies in place, optimiser steps, init_weights), data pointers on re-allocation (.to())
    stamp = tuple((v.data_ptr(), v._version) for v in sd.values())
    hit = _GENERATORS.get(id(net))
    if hit is None or hit[1] != stamp:
        if hit is None:
            gen = HeadposeGenerator(opt, sd)
        else:
            gen = hit[0]
            gen.load_state_dict(sd)
        _GENERATORS.clear()
        _GENERATORS[id(net)] = (gen, stamp)
    gen = _GENERATORS[id(net)][0]
    audio = np.asarray(audio_feats, dtype=np.float32).reshape(-1, 512 * 2)              # :148
    nframe = audio.shape[0] - opt.frame_future
    if getattr(opt, "loss", "GMM") == "GMM":
        noise, uniform = draw_reference_noise(nframe, opt.A2H_GMM_ndim, opt.A2H_GMM_ncenter)
    else:
        noise, uniform = None, None
    pred = gen.generate(audio, np.asarray(pre_headpose, dtype=np.float32), noise, sigma_scale, uniform)
    return pred.cpu().numpy().astype(np.float64)                                        # :150 np.zeros default dtype


def install(models_module_name: str = "models.audio2headpose_model") -> None:
    """Swap the reference's loop for the CUDA one; ``demo.py`` then runs unchanged (demo.py:212)."""
    import importlib
    mod = importlib.import_module(models_module_name)
    mod.Audio2HeadposeModel.generate_sequences = generate_sequences
