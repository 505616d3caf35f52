"""Log-mel front end on the GPU (SURVEY.md 8f, row N6): a drop-in for ``compute_mel_one_sequence`` (funcs/utils.py:61-83),
stage 1 of ``demo.py`` (:185).

The reference loops over the ``2 nframe`` windows of the clip in Python; each iteration sends a 266-sample clip to the
device, runs ``Audio2Mel.forward`` (reflect pad, one ``torch.stft`` frame, magnitude, mel matmul, log) and copies the 80
values back.  ``MelFrontEnd.logmel`` computes every window in one kernel (include/lspa.h, csrc/lspa.cu) and leaves the
result on the device, so the chain audio -> log-mel -> APC GRU -> ``ManifoldProjector`` -> ``HeadposeGenerator`` needs no
host round trip.  The mel filterbank is an input: ``mel_basis()`` gives librosa's where librosa is installed and a
numpy restatement of it otherwise.

``install()`` patches ``compute_mel_one_sequence`` of the reference's ``funcs.utils`` module; ``demo.py`` calls it as a
module attribute, so it then runs unchanged.  There is no CPU path.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np
import torch

from . import _lib

N_FFT = 512
N_BINS = N_FFT // 2 + 1
MAX_MELS = 128
FRAME_LEN_RANGE = (190, 266)   # Audio2Mel's reflect pad of 189 needs a longer clip, its single stft frame a shorter one


# ------------------------------------------------------------------------------------------------------------------
# The filterbank
# ------------------------------------------------------------------------------------------------------------------
_MIN_LOG_MEL = 1000.0 / (200.0 / 3)   # the mel of 1 kHz, where the Slaney scale turns logarithmic
_LOG_STEP = np.log(6.4) / 27.0


def _hz_to_mel(f):
    f = np.asarray(f, np.float64)
    log_t = f >= 1000.0
    return np.where(log_t, _MIN_LOG_MEL + np.log(np.where(log_t, f, 1000.0) / 1000.0) / _LOG_STEP, f / (200.0 / 3))


def _mel_to_hz(m):
    m = np.asarray(m, np.float64)
    return np.where(m >= _MIN_LOG_MEL, 1000.0 * np.exp(_LOG_STEP * (m - _MIN_LOG_MEL)), (200.0 / 3) * m)


def mel_band_edges(sr: int = 16000, n_mels: int = 80, fmin: float = 90.0, fmax: float = 7600.0) -> np.ndarray:
    """The ``n_mels + 2`` triangle edges in Hz: equally spaced on the Slaney mel scale (linear at 200/3 Hz per mel below
    1 kHz, logarithmic with step log(6.4) / 27 above) from fmin to fmax."""
    return _mel_to_hz(np.linspace(_hz_to_mel(fmin), _hz_to_mel(fmax), n_mels + 2))


def slaney_mel(sr: int = 16000, n_fft: int = 512, n_mels: int = 80, fmin: float = 90.0, fmax: float = 7600.0) -> np.ndarray:
    """``librosa.filters.mel`` as librosa 0.7.0 computes it (``htk=False``, ``norm=1``): fp32 [n_mels, 1 + n_fft // 2].
    Band i is the triangle over FFT bin frequencies rising from edge i to 1 at edge i + 1 and falling to 0 at edge
    i + 2, scaled by 2 / (edge[i + 2] - edge[i]) so that every band has the same area.  Not compared with librosa
    itself here (it is not a dependency)."""
    fft_f = np.linspace(0.0, float(sr) / 2, 1 + n_fft // 2, endpoint=True)
    edges = mel_band_edges(sr, n_mels, fmin, fmax)
    fdiff = np.diff(edges)
    ramps = np.subtract.outer(edges, fft_f)
    w = np.zeros((n_mels, fft_f.shape[0]), np.float32)
    for i in range(n_mels):
        w[i] = np.maximum(0, np.minimum(-ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]))
    w *= (2.0 / (edges[2:n_mels + 2] - edges[:n_mels]))[:, None]
    return w


def mel_basis(sr: int = 16000, n_fft: int = 512, n_mels: int = 80, fmin: float = 90.0, fmax: float = 7600.0) -> np.ndarray:
    """``Audio2Mel.mel_basis``: ``librosa.filters.mel`` when librosa imports, else ``slaney_mel``; fp32."""
    try:
        import librosa
    except ImportError:
        return slaney_mel(sr, n_fft, n_mels, fmin, fmax)
    return np.asarray(librosa.filters.mel(sr=sr, n_fft=n_fft, n_mels=n_mels, fmin=fmin, fmax=fmax), np.float32)


_default_basis = mel_basis   # MelFrontEnd's argument of the same name shadows it


def frame_len_of(sr, winlen) -> int:
    """``int(sr * winlen)`` (funcs/utils.py:71), refused with ``ValueError`` outside the range the reference runs in."""
    frame_len = int(sr * winlen)
    lo, hi = FRAME_LEN_RANGE
    if not lo <= frame_len <= hi:
        raise ValueError(f"frame length int(sr * winlen) = {frame_len} is outside [{lo}, {hi}]: Audio2Mel's reflect pad "
                         f"needs more than 189 samples and its stft must yield exactly one frame")
    return frame_len


# ------------------------------------------------------------------------------------------------------------------
# The device front end
# ------------------------------------------------------------------------------------------------------------------
class MelFrontEnd:
    """Owns the native handle and a device copy of the mel basis (fp32 [n_mels, 257], 1 <= n_mels <= 128; ``mel_basis()``
    by default).  The copy is taken at construction."""

    def __init__(self, mel_basis=None, device: Optional[torch.device] = None):
        self._lib = _lib.load()
        self._handle = C.c_void_p()
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("livespeechportraits_b200 has no CPU path: the log-mel front end needs an H100 (sm_90) device")
        self.device = device if device.index is not None else torch.device("cuda", torch.cuda.current_device())
        basis = _default_basis() if mel_basis is None else mel_basis
        if isinstance(basis, torch.Tensor):
            basis = basis.detach().cpu().numpy()
        basis = np.ascontiguousarray(basis, dtype=np.float32)
        if basis.ndim != 2 or basis.shape[1] != N_BINS or not 1 <= basis.shape[0] <= MAX_MELS:
            raise ValueError(f"mel_basis must be [n_mels <= {MAX_MELS}, {N_BINS}], got shape {basis.shape}")
        self.n_mels = basis.shape[0]
        _lib.check_a(self._lib.lspa_create(C.byref(self._handle), self.device.index))
        _lib.check_a(self._lib.lspa_load_mel_basis(self._handle, basis.ctypes.data, self.n_mels, N_BINS))

    def logmel(self, audio, winlen: float = 1 / 60, winstep: float = 0.5 / 60, sr: int = 16000,
               normalize: bool = True) -> torch.Tensor:
        """The log-mel frames of ``audio`` (1-D; numpy or torch, any float dtype, any device; rounded to fp32 as the
        reference's ``.float()`` does): CUDA fp32 [2 nframe, n_mels] with ``nframe = int(len(audio) / 16000 * 60)``,
        window i starting at ``int(i * sr * winstep)``.  Enqueued on the current stream; no host synchronisation."""
        frame_len = frame_len_of(sr, winlen)
        step = float(sr * winstep)
        a = torch.as_tensor(audio)
        if a.dim() != 1:
            raise ValueError(f"audio must be 1-D, got shape {tuple(a.shape)}")
        a = a.to(device=self.device, dtype=torch.float32).contiguous()
        n = 2 * int(a.shape[0] / 16000 * 60)
        out = torch.empty((n, self.n_mels), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device).cuda_stream
            _lib.check_a(self._lib.lspa_logmel(self._handle, a.data_ptr() if a.numel() else None, a.shape[0], n, frame_len,
                                               step, int(bool(normalize)), out.data_ptr() if n else None, stream))
        return out

    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                self._lib.lspa_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass


def compute_mel_one_sequence(audio, hop_length=int(16000 / 120), winlen=1 / 60, winstep=0.5 / 60, sr=16000, fps=60,
                             device='cpu'):   # noqa: N802 - reference name and signature
    """Replacement for funcs/utils.py ``compute_mel_one_sequence`` (:61-83): same arguments, same result (float64 numpy
    [2 nframe, 80] holding fp32 values).  ``hop_length``, ``fps`` and ``device`` do not change the numbers, as in the
    reference; the work runs on the current CUDA device whatever ``device`` says.  Raises ``ValueError`` for a frame length
    the reference cannot process, before any device work."""
    frame_len_of(sr, winlen)
    front = MelFrontEnd()                        # the basis is uploaded on every call: nothing is cached across calls
    return front.logmel(np.asarray(audio), winlen=winlen, winstep=winstep, sr=sr).cpu().numpy().astype(np.float64)


def install(module_name: str = "funcs.utils") -> None:
    """Swap the reference's ``compute_mel_one_sequence`` for the CUDA one; ``demo.py`` then runs unchanged (it calls it
    as ``utils.compute_mel_one_sequence``, demo.py:185)."""
    import importlib
    mod = importlib.import_module(module_name)
    mod.compute_mel_one_sequence = compute_mel_one_sequence
