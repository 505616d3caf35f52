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


class _Recurrent(_lib.Handle):
    """Owns one native handle (packed weights on one device)."""
    prefix = "lspr"

    def __init__(self, cfg: _lib.LsprConfig, state_dict: Dict[str, torch.Tensor], device):
        super().__init__(device)
        self.cfg = cfg
        self._create(C.byref(cfg))
        self.load_state_dict(state_dict)

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor]) -> None:
        arr, _keep = _lib.tensor_array(state_dict)
        self.call("load_weights", arr, len(arr))

    def packed(self, which: int) -> np.ndarray:
        """The array ``lspr_debug_packed`` returns (see include/lspr.h for the order)."""
        n = C.c_int64()
        self.call("debug_packed", which, None, C.byref(n))
        out = np.empty(n.value, np.float32)
        self.call("debug_packed", which, out.ctypes.data, C.byref(n))
        return out

    def _input(self, x: torch.Tensor, width: int) -> torch.Tensor:
        if not isinstance(x, torch.Tensor) or not x.is_cuda:
            raise RuntimeError("input must be a CUDA tensor (there is no CPU path)")
        if self.device is None:
            raise RuntimeError("host-only handle: created with device=-1")
        if x.dim() != 2 or x.shape[1] != width:
            raise ValueError(f"input must be [n, {width}], got {tuple(x.shape)}")
        x = x.to(device=self.device, dtype=torch.float32).contiguous()
        return x.clone() if x.data_ptr() % 16 else x

    def _new_state(self) -> torch.Tensor:
        """Uninitialised: the call from step 0 zeroes it."""
        if self.device is None:
            raise RuntimeError("host-only handle: created with device=-1")
        need = C.c_size_t()
        self.call("state_bytes", C.byref(need))
        return torch.empty(need.value // 4, dtype=torch.float32, device=self.device)

    def _run(self, x: torch.Tensor, step0: int, state: torch.Tensor, ws, n_out: int, out_dim: int, cluster: int):
        """One ``lspr_forward_stream`` call: ``x`` [n, width] from global step ``step0``, with the workspace ``ws``
        (None, or grown if too small); returns ([n_out, out_dim], the workspace)."""
        n = x.shape[0]
        out = torch.empty((n_out, out_dim), dtype=torch.float32, device=self.device)
        ws = _lib.reserve(ws, self.workspace_bytes(n), self.device)
        with self.cuda_stream() as stream:
            self.call("forward_stream", x.data_ptr() if n else None, n, int(step0), out.data_ptr() if n_out else None,
                      state.data_ptr(), ws.data_ptr(), ws.numel(), int(cluster), stream)
        self._keep = (x, state, ws)    # the buffers stay alive until the caller synchronises on the result
        return out, ws


class ApcEncoder(_Recurrent):
    """``APC_encoder`` on one clip.  ``state_dict`` uses its key grammar (``rnns.{i}.weight_ih_l0``, ...; an optional
    ``module.`` prefix is accepted); the layer count and mel width are read from it.  ``device=-1`` makes a host-only
    handle (packing introspection)."""
    what = "the APC encoder"

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
        x = self._input(mel, self.mel_dim)
        return self._run(x, 0, self._new_state(), None, x.shape[0], self.hidden, cluster)[0]

    __call__ = forward

    def stream(self, cluster: int = 0) -> "ApcStream":
        """A stream over one clip's mel frames: ``push(mel)`` returns the features of the rows pushed, and the
        concatenation equals ``forward`` of all of them, bit for bit."""
        return ApcStream(self, cluster)


class ApcStream:
    """The APC encoder over a clip pushed in pieces (``ApcEncoder.stream``).  Keeps each layer's last h and a workspace
    sized for the largest push so far on the device; every push is enqueued on the current stream with no host
    synchronisation (the pushes of one stream reuse the workspace, so they go on one CUDA stream)."""

    def __init__(self, enc: ApcEncoder, cluster: int = 0):
        self._enc, self._cluster = enc, int(cluster)
        self._state = enc._new_state()
        self._ws = None                        # workspace, kept across pushes
        self.rows = 0                          # mel frames pushed so far

    def push(self, mel: torch.Tensor) -> torch.Tensor:
        """mel [n, mel_dim] CUDA (n >= 0) -> features [n, hidden] CUDA fp32."""
        x = self._enc._input(mel, self._enc.mel_dim)
        out, self._ws = self._enc._run(x, self.rows, self._state, self._ws, x.shape[0], self._enc.hidden, self._cluster)
        self.rows += x.shape[0]
        return out

    def finish(self) -> torch.Tensor:
        """Nothing is held back: an empty [0, hidden] tensor."""
        return torch.empty((0, self._enc.hidden), dtype=torch.float32, device=self._enc.device)


def mouth_output_size(opt) -> int:
    """models/audio2feature.py:11-15."""
    if getattr(opt, "loss", "L2") == "GMM":
        return (2 * int(opt.A2L_GMM_ndim) + 1) * int(opt.A2L_GMM_ncenter)
    return int(opt.A2L_GMM_ndim) * int(getattr(opt, "predict_length", 1))


class MouthGenerator(_Recurrent):
    """Audio2Mouth: ``Audio2Feature`` with ``feature_decoder='LSTM'`` as ``generate_sequences`` runs it.  ``state_dict``
    uses its key grammar (``downsample.0.weight``, ``LSTM.weight_ih_l0``, ``fc.1.running_var``, ...)."""
    what = "Audio2Mouth"

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
        x = self._input(feats, self.apc_hidden)
        x = torch.cat([x, x[-1:].expand(2 * self.frame_future, -1)])    # models/audio2feature_model.py:134
        return self._run(x, 0, self._new_state(), None, n // 2, self.out_dim, 0)[0]

    def stream(self) -> "MouthStream":
        """A stream over one clip's APC features: ``push(feats)`` returns the track rows whose inputs are all in (frame f
        needs APC rows up to 2 (f + frame_future) + 1), ``finish()`` the last ``frame_future`` rows, built from copies of
        the last APC row.  The concatenation equals ``generate`` of all the rows, bit for bit."""
        return MouthStream(self)


class MouthStream:
    """Audio2Mouth over a clip pushed in pieces (``MouthGenerator.stream``).  Keeps the LSTM's h and c, one pending odd
    APC row, the last APC row and a workspace sized for the largest push so far on the device; every call is enqueued on
    the current stream with no host synchronisation (one CUDA stream per stream object, as the workspace is reused)."""

    def __init__(self, gen: MouthGenerator):
        self._gen = gen
        self._state = gen._new_state()
        self._ws = None                        # workspace, kept across pushes
        self._odd = None                       # an APC row waiting for its pair
        self._last = None                      # the last APC row: finish() pads with copies of it
        self.pairs = 0                         # LSTM steps run so far
        self.frames = 0                        # track rows returned so far
        self.finished = False

    def _run(self, x: torch.Tensor) -> torch.Tensor:
        ff, np_ = self._gen.frame_future, x.shape[0] // 2
        n_out = max(0, self.pairs + np_ - max(self.pairs, ff))          # the new global steps >= frame_future
        out, self._ws = self._gen._run(x, self.pairs, self._state, self._ws, n_out, self._gen.out_dim, 0)
        self.pairs += np_
        self.frames += n_out
        return out

    def push(self, feats: torch.Tensor) -> torch.Tensor:
        """APC features [n, APC_hidden] CUDA (any n >= 0) -> the new track rows [m, out_dim], frames
        ``frames - m .. frames - 1``."""
        if self.finished:
            raise RuntimeError("the stream has finished")
        x = self._gen._input(feats, self._gen.apc_hidden)
        if x.shape[0]:
            self._last = x[-1:].clone()
        if self._odd is not None:
            x = torch.cat([self._odd, x])
        even = x.shape[0] // 2 * 2
        self._odd = x[even:].clone() if even < x.shape[0] else None
        return self._run(x[:even])

    def finish(self) -> torch.Tensor:
        """The last ``frame_future`` track rows (fewer if the clip had fewer pairs; none for an empty clip)."""
        if self.finished:
            raise RuntimeError("the stream has finished")
        self.finished = True
        if self._odd is not None:
            n = 2 * self.pairs + 1
            raise RuntimeError(f"shape '[1, -1, {2 * self._gen.apc_hidden}]' is invalid for input of size "
                               f"{(n + 2 * self._gen.frame_future) * self._gen.apc_hidden}")
        if self.pairs == 0 or self._gen.frame_future == 0:
            return torch.empty((0, self._gen.out_dim), dtype=torch.float32, device=self._gen.device)
        return self._run(self._last.expand(2 * self._gen.frame_future, -1).contiguous())


# ------------------------------------------------------------------------------------------------------------------
# Drop-ins for the reference modules
# ------------------------------------------------------------------------------------------------------------------
_APC: "Dict[int, tuple]" = {}          # id(module) -> (ApcEncoder, stamp)
_MOUTH: "Dict[int, tuple]" = {}        # id(module) -> (MouthGenerator, stamp)


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
    enc = _lib.cached(_APC, self, lambda sd: ApcEncoder(sd, inputs.device, residual=bool(self.rnn_residual)),
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
    gen = _lib.cached(_MOUTH, net, make, (ff, str(device)))
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
