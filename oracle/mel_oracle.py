"""Oracle of the log-mel front end (SURVEY.md 8f row N6): ``compute_mel_one_sequence`` (funcs/utils.py:61-83) and
``Audio2Mel.forward`` (funcs/audio_funcs.py:56-75), stage 1 of demo.py (:185).  TEST INFRASTRUCTURE.

Restated with the same torch calls and dtypes on the CPU (nothing is copied):

* ``compute_mel_one_sequence``  <- the per-window loop: ``nframe = int(len / 16000 * 60)``, ``2 nframe`` windows starting
                                   at ``int(i * sr * winstep)``, each ``audio[st:st+L]`` zero-padded to
                                   ``L = int(sr * winlen)`` and rounded to fp32
* ``audio2mel``                 <- ``Audio2Mel(n_fft=512, hop_length=133, win_length=266, ...)``: reflect pad of 189 on
                                   each side of the clip, one ``torch.stft(center=False)`` frame with the periodic
                                   ``hann_window(266)`` centred in 512, ``sqrt(re^2 + im^2)``, ``mel_basis @ mag``,
                                   ``log(clamp(., 1e-5))`` and ``(x - m) / -m`` with ``m = log(1e-5)``

``torch.stft`` without ``return_complex`` is refused by torch >= 2; the restatement asks for the complex result and takes
``view_as_real`` of it, which is the real [.., 2] layout torch 1.7 returned.  The mel basis is an input everywhere: the
reference builds it with ``librosa.filters.mel``; ``slaney_mel`` (livespeechportraits_b200/audio.py) restates that
(librosa 0.7.0, ``htk=False``, area normalisation) for machines without librosa.  librosa is not installed where this
oracle was written, so the restatement is pinned by its structural facts only (tests/test_mel_oracle.py), not against
librosa itself.

``logmel_truth`` is the float64 truth the CUDA kernel is judged by: the same fp32 clip and the exact Hann window in
float64, ``np.fft.rfft``, a float64 product with the (fp32) basis and a float64 log.
"""
from __future__ import annotations

import ast
import math
import os
import types
from typing import Optional

import numpy as np
import torch
import torch.nn.functional as F

REFERENCE_ROOT = os.environ.get("LSP_REFERENCE_ROOT", "/root/reference")
UTILS_FILE = os.path.join(REFERENCE_ROOT, "funcs", "utils.py")
AUDIO_FUNCS_FILE = os.path.join(REFERENCE_ROOT, "funcs", "audio_funcs.py")
WAV_FILE = os.path.join(REFERENCE_ROOT, "data", "Input", "00083.wav")

SR = 16000
N_FFT = 512
HOP = int(16000 / 120)            # 133: Audio2Mel's hop, which sets the reflect pad
WIN = int(16000 / 60)             # 266: Audio2Mel's window, whatever winlen the caller passes
N_BINS = N_FFT // 2 + 1           # 257
PAD = (N_FFT - HOP) // 2          # 189
WIN_OFFSET = (N_FFT - WIN) // 2   # 123: torch.stft centres a short window in n_fft
MIN_LEVEL = 1e-5
MIN_MEL = math.log(MIN_LEVEL)
FRAME_LEN_RANGE = (PAD + 1, WIN)  # the reflect pad needs PAD < L; one stft frame needs L + 2 PAD - n_fft < hop


def n_windows(n_samples: int) -> int:
    """``2 * int(len(audio) / 16000 * 60)`` with the literal constants of funcs/utils.py:67."""
    return 2 * int(n_samples / 16000 * 60)


def window_starts(n: int, step: float) -> np.ndarray:
    """``int(i * step)`` for i < n: the float64 product truncated, as funcs/utils.py:74 forms it."""
    return np.array([int(i * step) for i in range(n)], dtype=np.int64)


def clip(audio: np.ndarray, st: int, frame_len: int) -> np.ndarray:
    """``audio[st:st+L]`` zero-padded at the end to L, rounded to fp32 (funcs/utils.py:75-78)."""
    c = np.zeros(frame_len, np.float32)
    seg = np.asarray(audio[st:st + frame_len]).astype(np.float32)
    c[:seg.shape[0]] = seg
    return c


# ------------------------------------------------------------------------------------------------------------------
# The mel filterbank
# ------------------------------------------------------------------------------------------------------------------
# ``slaney_mel`` lives in the package (``mel_basis()`` falls back to it where librosa is missing); it is an input of the
# kernel, not something the kernel computes, so the oracle uses the same function.
from livespeechportraits_b200.audio import mel_band_edges, slaney_mel  # noqa: E402,F401


def make_basis(n_mels: int = 80, seed: Optional[int] = None) -> np.ndarray:
    """The Slaney basis, or (seed given) a random non-negative fp32 basis of the same shape, so that a test does not
    depend on the filterbank's shape."""
    if seed is None:
        return slaney_mel(n_mels=n_mels)
    rng = np.random.Generator(np.random.PCG64(seed))
    return (rng.random((n_mels, N_BINS)) * 0.05).astype(np.float32)


# ------------------------------------------------------------------------------------------------------------------
# Restatement of the reference (fp32, same calls)
# ------------------------------------------------------------------------------------------------------------------
def normalize_fp32(x):
    """``(x - m) / -m`` as torch evaluates it on an fp32 CPU tensor: the Python float m is rounded to fp32, then an fp32
    subtraction and an fp32 division (evaluating in float64 and rounding once gives different values).  fp32 in, out."""
    x = np.asarray(x, np.float32)
    m = np.float32(MIN_MEL)
    return (x - m) / -m


def _stft_real(x, **kw):
    return torch.view_as_real(torch.stft(x, return_complex=True, **kw))


def audio2mel(clips: torch.Tensor, mel_basis: torch.Tensor, normalize: bool = True) -> torch.Tensor:
    """``Audio2Mel.forward`` (funcs/audio_funcs.py:56-75) on fp32 ``clips`` [B, 1, L]; returns [B, n_mels, 1]."""
    p = (N_FFT - HOP) // 2
    audio = F.pad(clips, (p, p), "reflect").squeeze(1)
    fft = _stft_real(audio, n_fft=N_FFT, hop_length=HOP, win_length=WIN, window=torch.hann_window(WIN).float().to(clips.device),
                     center=False)
    real_part, imag_part = fft.unbind(-1)
    magnitude = torch.sqrt(real_part ** 2 + imag_part ** 2)
    mel_output = torch.matmul(mel_basis, magnitude)
    log_mel_spec = torch.log(torch.clamp(mel_output, min=MIN_LEVEL))
    if normalize:
        log_mel_spec = (log_mel_spec - MIN_MEL) / -MIN_MEL
    return log_mel_spec


def compute_mel_one_sequence(audio: np.ndarray, mel_basis: np.ndarray, winlen: float = 1 / 60, winstep: float = 0.5 / 60,
                             sr: int = 16000, normalize: bool = True, batched: bool = False) -> np.ndarray:
    """funcs/utils.py:61-83 with the given basis: float64 [2 nframe, n_mels] holding fp32 values.  ``batched`` runs all
    windows through one ``audio2mel`` call (same values up to the batched matmul's summation order; for long clips)."""
    nframe = int(audio.shape[0] / 16000 * 60)
    frame_len = int(sr * winlen)
    step = sr * winstep
    basis = torch.from_numpy(np.ascontiguousarray(mel_basis, np.float32))
    out = np.zeros([2 * nframe, basis.shape[0]])
    starts = window_starts(2 * nframe, step)
    if batched and nframe:
        clips = torch.from_numpy(np.stack([clip(audio, int(st), frame_len) for st in starts]))[:, None, :]
        for b0 in range(0, clips.shape[0], 4096):
            out[b0:b0 + 4096] = audio2mel(clips[b0:b0 + 4096], basis, normalize)[..., 0].numpy()
        return out
    for i, st in enumerate(starts):
        c = torch.from_numpy(clip(audio, int(st), frame_len))[None, None, :]
        out[i] = audio2mel(c, basis, normalize).numpy()[0].T
    return out


# ------------------------------------------------------------------------------------------------------------------
# float64 truth
# ------------------------------------------------------------------------------------------------------------------
def frames64(audio: np.ndarray, windows: np.ndarray, frame_len: int = WIN, step: float = SR * 0.5 / 60) -> np.ndarray:
    """[len(windows), 512] float64: the exact periodic Hann window times the reflect-padded fp32 clip of each window
    index, at its place in the frame."""
    idx = np.arange(WIN_OFFSET, WIN_OFFSET + WIN) - PAD           # position in the clip before reflection
    idx = np.where(idx < 0, -idx, idx)
    idx = np.where(idx >= frame_len, 2 * (frame_len - 1) - idx, idx)
    hann = 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(WIN) / WIN)
    a32 = np.concatenate([np.asarray(audio).astype(np.float32), np.zeros(frame_len, np.float32)])
    out = np.zeros((len(windows), N_FFT))
    for r, i in enumerate(windows):
        st = min(int(int(i) * step), a32.shape[0] - frame_len)     # past the end: zeros either way
        out[r, WIN_OFFSET:WIN_OFFSET + WIN] = hann * a32[st:st + frame_len].astype(np.float64)[idx]
    return out


def logmel_truth(audio: np.ndarray, mel_basis: np.ndarray, windows: Optional[np.ndarray] = None, frame_len: int = WIN,
                 step: float = SR * 0.5 / 60, normalize: bool = True) -> dict:
    """float64 log-mel of the given windows (all ``n_windows(len(audio))`` by default) and the quantities the error bound
    of the CUDA kernel is made of: ``out`` [n, M], ``mel`` [n, M] (before the clamp) and ``bmag`` [n, M] =
    sum_k B[m, k] (|X_k| + S) with S = sum_t |w_t x_t| the frame's l1 mass."""
    if windows is None:
        windows = np.arange(n_windows(audio.shape[0]))
    fr = frames64(audio, windows, frame_len, step)
    mag = np.abs(np.fft.rfft(fr, axis=1))
    B = np.asarray(mel_basis, np.float64)
    mel = mag @ B.T
    lg = np.log(np.maximum(mel, MIN_LEVEL))
    out = (lg - MIN_MEL) / -MIN_MEL if normalize else lg
    bmag = mel + np.abs(fr).sum(1, keepdims=True) * B.sum(1)[None, :]
    return {"out": out, "mel": mel, "bmag": bmag}


def error_bound(t: dict, normalize: bool = True) -> np.ndarray:
    """Per-element bound on |kernel - float64 truth| for csrc/lspa.cu's arithmetic (u = 2^-24, fp32 throughout):

    1. frame: w_t fp32 (|dw| <= u w), x_t exact, product rounded: |d(w x)| <= 2.01 u |w x|.
    2. DFT: 266 fma terms per part, summed in order, twiddles rounded once from fp64 (|dc| <= u): each of re and im is
       off by at most (266 + 3) u S with S = sum_t |w_t x_t|, so |d mag| <= sqrt(2) 269 u S + the sqrt and the squares
       (3 u |X|): e_k = 381 u S + 3 u |X_k|.
    3. mel: sum_k B_mk mag_k in 257 fma steps (B exact): |d mel| <= sum_k B_mk e_k + 258 u sum_k B_mk (|X_k| + e_k)
       <= 640 u sum_k B_mk (|X_k| + S) = 640 u bmag (second-order terms absorbed by the rounding of 381 up).
    4. log of the clamp: with d = |d mel|, |d log| <= d / max(mel - d, 1e-5) (the clamp is 1-Lipschitz in log terms,
       and a mel below 1e-5 on both sides gives log(1e-5f)), plus logf's 2 ulp of |log| (<= 2 u * 16 for |log| <= 16).
    5. normalise: (x - m) * (1 / -m) in fp32: |d| <= (|d log| + u |x - m|) / |m| + 2 u |out| + u |out|.
    """
    u = 2.0 ** -24
    d = 640.0 * u * t["bmag"]
    mel = t["mel"]
    dlog = d / np.maximum(mel - d, MIN_LEVEL) + 32.0 * u
    if not normalize:
        return dlog
    lg = t["out"] * -MIN_MEL + MIN_MEL
    return (dlog + u * np.abs(lg - MIN_MEL)) / -MIN_MEL + 3.0 * u * np.abs(t["out"]) + 1e-12


# ------------------------------------------------------------------------------------------------------------------
# The APC encoder in front of the manifold projection
# ------------------------------------------------------------------------------------------------------------------
class ApcGru(torch.nn.Module):
    """``APC_encoder`` (models/networks.py) as demo.py runs it on one clip: a stack of single-layer GRUs (mel 80 -> 512,
    then 512 -> 512), each layer's output plus its input where the widths match (residual), the last layer's output
    returned.  ``pack_padded_sequence`` with the full length is the identity, so it is left out.  Weights are torch's
    default initialisation under ``seed``."""

    def __init__(self, mel_dim: int = 80, hidden: int = 512, layers: int = 3, seed: int = 0):
        super().__init__()
        with torch.random.fork_rng(devices=[]):
            torch.manual_seed(seed)
            sizes = [mel_dim] + [hidden] * layers
            self.rnns = torch.nn.ModuleList([torch.nn.GRU(sizes[i], sizes[i + 1], batch_first=True) for i in range(layers)])

    @torch.no_grad()
    def forward(self, mel: torch.Tensor) -> torch.Tensor:
        """mel [T, mel_dim] -> features [T, hidden]."""
        x = mel[None]
        for i, rnn in enumerate(self.rnns):
            y = rnn(x)[0]
            if i + 1 < len(self.rnns) and y.shape[-1] == x.shape[-1]:
                y = y + x
            x = y
        return x[0]


# ------------------------------------------------------------------------------------------------------------------
# Test audio
# ------------------------------------------------------------------------------------------------------------------
def make_audio(n_samples: int, seed: int = 0) -> np.ndarray:
    """Deterministic fp32 test audio in [-1, 1], in segments of 2000 samples cycling through: a linear chirp (amplitude 0.3) 100 Hz ->
    7.9 kHz, white noise, exact silence, a clipped tone over noise (+-1 exactly on its peaks), low-level noise (-60 dB) and a
    chirp over noise.  Every loud segment carries -30 dB of noise, so that no band of a loud window sits at the fp32
    noise floor of the DFT, where the reference's own fp32 result is off by more than 1e-5."""
    rng = np.random.Generator(np.random.PCG64(seed))
    t = np.arange(n_samples) / SR
    seg = (np.arange(n_samples) // 2000) % 6
    ph = (t % 0.125) / 0.125
    chirp = np.sin(2 * np.pi * (100.0 * ph * 0.125 + 0.5 * (7800.0 / 0.125) * (ph * 0.125) ** 2))
    noise = rng.random(n_samples) * 2.0 - 1.0
    floor = 3e-2 * (rng.random(n_samples) * 2.0 - 1.0)
    clipped = np.clip(1.5 * np.sin(2 * np.pi * 440.0 * t), -1.0, 1.0)
    x = np.select([seg == 0, seg == 1, seg == 2, seg == 3, seg == 4, seg == 5],
                  [0.3 * chirp + floor, 0.5 * noise, 0.0 * t, np.clip(clipped + floor, -1.0, 1.0), 0.03 * floor,
                   0.3 * chirp + 0.1 * noise])
    return np.clip(x, -1.0, 1.0).astype(np.float32)


def read_wav(path: str = WAV_FILE) -> np.ndarray:
    """The shipped clip as demo.py's ``librosa.load(sr=16000)`` would return it: the file is already 16 kHz mono fp32,
    so ``scipy.io.wavfile`` gives the samples directly (that librosa returns the same samples is assumed here)."""
    from scipy.io import wavfile
    sr, a = wavfile.read(path)
    assert sr == SR and a.dtype == np.float32 and a.ndim == 1, (sr, a.dtype, a.shape)
    return a


def read_wav_fixture() -> np.ndarray:
    """The 00083.wav samples as stored in tests/golden/mel/ (machines without the reference checkout)."""
    here = os.path.dirname(os.path.abspath(__file__))
    return np.load(os.path.join(os.path.dirname(here), "tests", "golden", "mel", "mel_00083_wav.npz"))["audio"]


# ------------------------------------------------------------------------------------------------------------------
# The live reference (only where the reference checkout exists)
# ------------------------------------------------------------------------------------------------------------------
def reference_available() -> bool:
    return os.path.isfile(UTILS_FILE) and os.path.isfile(AUDIO_FUNCS_FILE)


class _TorchShim(types.ModuleType):
    """``torch`` with one change: ``stft`` asks for the complex result and returns ``view_as_real`` of it, the real
    [.., 2] layout the reference's torch 1.7 call returned (torch >= 2 refuses the call without ``return_complex``)."""

    def __init__(self):
        super().__init__("torch")

    def __getattr__(self, name):
        return getattr(torch, name)

    @staticmethod
    def stft(*args, **kw):
        return _stft_real(*args, **kw)


def reference_functions(mel_basis: np.ndarray) -> dict:
    """``compute_mel_one_sequence`` (funcs/utils.py) and ``Audio2Mel`` (funcs/audio_funcs.py) lifted out with ``ast`` and
    executed unchanged (both modules import librosa).  ``librosa_mel_fn`` is a stub returning ``mel_basis``; ``torch``
    is ``_TorchShim``."""
    import warnings
    basis = np.ascontiguousarray(mel_basis, np.float32)
    ns: dict = {"np": np, "torch": _TorchShim(), "F": F, "math": math,
                "librosa_mel_fn": lambda sr, n_fft, n_mels, fmin, fmax: basis}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", SyntaxWarning)
        for path, wanted in ((AUDIO_FUNCS_FILE, ("Audio2Mel",)), (UTILS_FILE, ("compute_mel_one_sequence",))):
            tree = ast.parse(open(path).read())
            nodes = [nd for nd in tree.body if isinstance(nd, (ast.FunctionDef, ast.ClassDef)) and nd.name in wanted]
            assert sorted(nd.name for nd in nodes) == sorted(wanted), path
            exec(compile(ast.fix_missing_locations(ast.Module(body=nodes, type_ignores=[])), path, "exec"), ns)
            if "Audio2Mel" in wanted:
                ns["audio_funcs"] = types.SimpleNamespace(Audio2Mel=ns["Audio2Mel"])
    return {"compute_mel_one_sequence": ns["compute_mel_one_sequence"], "Audio2Mel": ns["Audio2Mel"]}
