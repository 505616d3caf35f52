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


class HeadposeGenerator(_lib.Handle):
    """Owns the native handle (packed weights on one device).  ``state_dict`` uses the key grammar of
    ``Audio2Headpose(opt).state_dict()`` (an optional ``module.`` prefix is accepted)."""
    prefix, what = "lsph", "the headpose loop"

    def __init__(self, opt, state_dict: Dict[str, torch.Tensor], device: Optional[torch.device] = None):
        self.cfg = config_from_opt(opt)
        super().__init__(device)
        self._create(C.byref(self.cfg))
        rf = C.c_int()
        self.call("receptive_field", C.byref(rf))
        self.receptive_field = rf.value
        self.out_channels = (2 * self.cfg.ndim + 1) * self.cfg.ncenter if self.cfg.loss_gmm else self.cfg.ndim
        self.load_state_dict(state_dict)

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor]) -> None:
        arr, _keep = _lib.tensor_array(state_dict)
        self.call("load_weights", arr, len(arr))

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
        for t in (a, pre, nz):
            if t.data_ptr() % 16:
                raise ValueError("device buffers must be 16-byte aligned")
        pred, params, _ = self._run(a, 0, 0, nframe, pre, nz, un, float(sigma_scale), self._new_state(), None, return_params,
                                    int(cluster))
        return (pred, params) if return_params else pred

    def _new_state(self) -> torch.Tensor:
        """A device buffer for the loop's state (include/lsph.h, ``lsph_state_bytes``); the call at frame 0 starts it."""
        need = C.c_size_t()
        self.call("state_bytes", C.byref(need))
        return torch.empty(need.value // 4, dtype=torch.float32, device=self.device)

    def _run(self, rows, row0: int, frame0: int, n: int, pre, noise, uniform, sigma_scale: float, state, ws,
             return_params: bool, cluster: int):
        """One ``lsph_generate_stream`` call: frames ``frame0 .. frame0 + n - 1`` from the device audio rows ``rows``
        (global rows ``row0 ..``; fp32, contiguous, 16-byte aligned) with the draws ``noise`` [n, ndim] and ``uniform``
        [n] (or None).  Returns pred [n, ndim], the network outputs [n, out_ch] (None without ``return_params``) and the
        workspace used (``ws`` or a larger one; nothing runs for n == 0)."""
        dev = self.device
        pred = torch.empty((n, self.cfg.ndim), dtype=torch.float32, device=dev)
        params = torch.empty((n, self.out_channels), dtype=torch.float32, device=dev) if return_params else None
        if n:
            need = C.c_size_t()
            self.call("stream_workspace_bytes", rows.shape[0], C.byref(need))
            ws = _lib.reserve(ws, need.value, dev)
            ptr = lambda t: t.data_ptr() if t is not None else None    # noqa: E731
            with self.cuda_stream() as stream:
                self.call("generate_stream", rows.data_ptr(), row0, rows.shape[0], frame0, n, pre.data_ptr(), ptr(noise),
                          ptr(uniform), sigma_scale, pred.data_ptr(), ptr(params), state.data_ptr(), ws.data_ptr(),
                          ws.numel(), cluster, stream)
            self._keep = (rows, pre, noise, uniform, state, ws)   # the buffers stay alive until the caller synchronises
        return pred, params, ws

    def stream(self, pre_headpose=None, sigma_scale: float = 0.3, noise=None, return_params: bool = False,
               cluster: int = 0) -> "HeadposeStream":
        """A stream over one clip's audio rows: ``push(rows)`` returns the frames whose look-ahead is in (frame i needs
        rows up to i + frame_future).  The concatenation equals ``generate`` of all the rows, bit for bit, given the same
        draws.  ``pre_headpose`` defaults to zeros (demo.py:211).  ``noise``: None draws each frame's ``Sample_GMM``
        values from torch's global CPU generator when the frame is produced, in ``draw_reference_noise``'s order (one
        mixture component only); or a callable ``noise(first_frame, n_frames)`` returning the draws of those frames,
        ``[n, ndim]`` or ``([n, ndim], uniform [n])``."""
        return HeadposeStream(self, pre_headpose, sigma_scale, noise, return_params, cluster)


class HeadposeStream:
    """The Audio2Headpose loop over a clip pushed in pieces (``HeadposeGenerator.stream``).  Keeps on the device the
    history ring and last sample (include/lsph.h, ``lsph_state_bytes``) and the audio rows not consumed yet - before the
    first frame, at most ``frame_future`` of them; afterwards none - and a workspace sized for the largest push so far.
    Pushes make no host synchronisation and, as they reuse the workspace, go on one CUDA stream."""

    def __init__(self, gen: HeadposeGenerator, pre_headpose, sigma_scale: float, noise, return_params: bool, cluster: int):
        if gen.device is None:
            raise RuntimeError("host-only handle: created with device=-1")
        cfg = gen.cfg
        if cfg.loss_gmm and noise is None and cfg.ncenter > 1:
            raise ValueError("with more than one mixture component the reference draws the component after the loop; "
                             "pass a noise callable that returns (noise, uniform)")
        self._gen, self._sigma, self._noise, self._params, self._cluster = gen, float(sigma_scale), noise, return_params, int(cluster)
        pre = torch.zeros(cfg.input_ch) if pre_headpose is None else pre_headpose
        self._pre = _lib.to_device(pre, gen.device).reshape(-1)
        if self._pre.numel() != cfg.input_ch:
            raise ValueError(f"pre_headpose must have {cfg.input_ch} values")
        self._state = gen._new_state()
        self._ws = None                        # workspace of the hoisted GEMMs, kept across pushes
        self._rows = torch.empty((0, 2 * cfg.apc_hidden), dtype=torch.float32, device=gen.device)
        self._row0 = 0                         # global index of self._rows[0]
        self.rows = 0                          # audio rows pushed so far
        self.frames = 0                        # frames returned so far

    def _draws(self, n: int):
        cfg = self._gen.cfg
        if not cfg.loss_gmm:
            return None, None
        if self._noise is None:
            noise, _ = draw_reference_noise(n, cfg.ndim, 1)
            uniform = None
        else:
            got = self._noise(self.frames, n)
            noise, uniform = got if isinstance(got, tuple) else (got, None)
        dev = self._gen.device
        noise = _lib.to_device(noise, dev).reshape(n, cfg.ndim)
        uniform = _lib.to_device(uniform, dev).reshape(n) if uniform is not None else None
        return noise, uniform

    def push(self, audio_rows):
        """Audio rows [n, 2*APC_hidden] (any n >= 0) -> the new frames: pred [m, ndim] CUDA fp32 (and the network outputs
        [m, out_ch] with ``return_params``), frames ``frames - m .. frames - 1``."""
        cfg, dev = self._gen.cfg, self._gen.device
        a = _lib.to_device(audio_rows, dev).reshape(-1, 2 * cfg.apc_hidden)
        self.rows += a.shape[0]
        rows = torch.cat([self._rows, a]) if self._rows.shape[0] else a
        if rows.data_ptr() % 16:
            rows = rows.clone()
        n = max(0, self.rows - cfg.frame_future) - self.frames
        noise, uniform = self._draws(n) if n else (None, None)
        pred, params, self._ws = self._gen._run(rows, self._row0, self.frames, n, self._pre, noise, uniform, self._sigma,
                                                self._state, self._ws, self._params, self._cluster)
        self.frames += n
        keep = self.frames + cfg.frame_future if self.frames else 0          # the first row a later frame reads
        drop = min(max(keep - self._row0, 0), rows.shape[0])
        self._rows = rows[drop:].clone()
        self._row0 += drop
        return (pred, params) if self._params else pred

    def finish(self):
        """Nothing is held back (the loop has no end padding): empty outputs."""
        pred = torch.empty((0, self._gen.cfg.ndim), dtype=torch.float32, device=self._gen.device)
        params = torch.empty((0, self._gen.out_channels), dtype=torch.float32, device=self._gen.device)
        return (pred, params) if self._params else pred


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
    gen = _lib.cached(_GENERATORS, net, lambda sd: HeadposeGenerator(opt, sd))
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
