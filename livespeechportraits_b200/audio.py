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

The step in front of it, ``librosa.load(path, sr=16000)`` (demo.py:179), is ``Resampler`` / ``load_wav``: the mono mix and
resampy's ``kaiser_best`` resampling of native-rate audio, whole clips and live (``Resampler.stream``), in one kernel.
"""
from __future__ import annotations

import functools
import math
from typing import Optional, Tuple

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
class MelFrontEnd(_lib.Handle):
    """Owns the native handle and a device copy of the mel basis (fp32 [n_mels, 257], 1 <= n_mels <= 128; ``mel_basis()``
    by default).  The copy is taken at construction."""
    prefix, what = "lspa", "the log-mel front end"

    def __init__(self, mel_basis=None, device: Optional[torch.device] = None):
        super().__init__(device)
        basis = _default_basis() if mel_basis is None else mel_basis
        if isinstance(basis, torch.Tensor):
            basis = basis.detach().cpu().numpy()
        basis = np.ascontiguousarray(basis, dtype=np.float32)
        if basis.ndim != 2 or basis.shape[1] != N_BINS or not 1 <= basis.shape[0] <= MAX_MELS:
            raise ValueError(f"mel_basis must be [n_mels <= {MAX_MELS}, {N_BINS}], got shape {basis.shape}")
        self.n_mels = basis.shape[0]
        self._create()
        self.call("load_mel_basis", basis.ctypes.data, self.n_mels, N_BINS)

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
        with self.cuda_stream() as stream:
            self.call("logmel_at", a.data_ptr() if a.numel() else None, 0, a.shape[0], 0, n, frame_len, step,
                      int(bool(normalize)), out.data_ptr() if n else None, stream)
        return out


    def stream(self, winlen: float = 1 / 60, winstep: float = 0.5 / 60, sr: int = 16000,
               normalize: bool = True) -> "MelStream":
        """A stream over one clip's samples: ``push(samples)`` returns the windows that became complete, ``finish()`` the
        rest.  The concatenation equals ``logmel`` of all the samples, bit for bit."""
        return MelStream(self, winlen, winstep, sr, normalize)


class MelStream:
    """The log-mel frames of a clip pushed in pieces (``MelFrontEnd.stream``).  Window i is returned by the push that
    completes its ``frame_len`` samples, once ``i < 2 int(n / 16000 * 60)`` for the n samples pushed so far
    (``stream.mel_windows``); the windows that reach into the end padding come out at ``finish()``.  Only the samples
    from the start of the next window on are kept on the device."""

    def __init__(self, front: MelFrontEnd, winlen: float, winstep: float, sr: int, normalize: bool):
        self._front = front
        self.frame_len = frame_len_of(sr, winlen)
        self.step = float(sr * winstep)
        if not self.step > 0:
            raise ValueError(f"the window step sr * winstep must be > 0 (got {self.step})")
        self._normalize = int(bool(normalize))
        self.samples = 0                       # samples pushed so far
        self.windows = 0                       # windows returned so far
        self.finished = False
        self._tail = torch.empty(0, dtype=torch.float32, device=front.device)   # samples tail0 .. samples - 1
        self._tail0 = 0

    def push(self, samples) -> torch.Tensor:
        """1-D samples (numpy or torch, any float dtype, any device; 16 kHz mono) -> the new windows [m, n_mels] CUDA."""
        if self.finished:
            raise RuntimeError("the stream has finished")
        a = _lib.to_device(samples, self._front.device)
        if a.dim() != 1:
            raise ValueError(f"samples must be 1-D, got shape {tuple(a.shape)}")
        self.samples += a.shape[0]
        buf = torch.cat([self._tail, a]) if self._tail.numel() else a
        return self._emit(buf, False)

    def finish(self) -> torch.Tensor:
        """The windows that need the end padding."""
        if self.finished:
            raise RuntimeError("the stream has finished")
        self.finished = True
        return self._emit(self._tail, True)

    def _emit(self, buf: torch.Tensor, finished: bool) -> torch.Tensor:
        from .stream import mel_windows
        ready = mel_windows(self.samples, finished, self.frame_len, self.step)
        k = ready - self.windows
        out = torch.empty((k, self._front.n_mels), dtype=torch.float32, device=self._front.device)
        if k:
            with self._front.cuda_stream() as stream:
                self._front.call("logmel_at", buf.data_ptr() if buf.numel() else None, self._tail0, buf.shape[0], self.windows,
                                 k, self.frame_len, self.step, self._normalize, out.data_ptr(), stream)
        self.windows = ready
        keep = min(int(self.windows * self.step), self.samples)        # where the next window starts
        self._tail = buf[keep - self._tail0:].clone()
        self._tail0 = keep
        self._keep = buf
        return out


# ------------------------------------------------------------------------------------------------------------------
# Resampling to 16 kHz: librosa.load's to_mono + resampy.resample (kaiser tables) + fix_length
# ------------------------------------------------------------------------------------------------------------------
SR = 16000
# resampy's shipped tables: num_zeros, precision (2^precision entries per zero crossing), Kaiser beta, rolloff
RESAMPLE_FILTERS = {"kaiser_best": (64, 9, 14.769656459379492, 0.9475937167399596),
                    "kaiser_fast": (16, 9, 8.555504641634386, 0.85)}
REGISTER_HORIZON = 1 << 40      # outputs the register table covers: about 2.2 years at 16 kHz


def resample_filter(name: str = "kaiser_best") -> Tuple[np.ndarray, int]:
    """resampy's half window (fp64 [num_zeros * num_table + 1]) and num_table for the filter ``name``: resampy's own
    table when resampy imports, else its ``sinc_window`` restated with ``scipy.signal.windows.kaiser``
    (``taper[n:] * rolloff * sinc(rolloff * linspace(0, num_zeros, n + 1))``, n = num_table * num_zeros), which may
    differ from the shipped ``.npz`` in the last bits.  The table is an input of ``Resampler``, like ``mel_basis``."""
    if name not in RESAMPLE_FILTERS:
        raise ValueError(f"unknown filter {name!r}; supported: {sorted(RESAMPLE_FILTERS)}")
    try:
        from resampy.filters import get_filter
    except ImportError:
        return _sinc_window(*RESAMPLE_FILTERS[name])
    win, num_table, _ = get_filter(name)
    return np.asarray(win, np.float64), int(num_table)


@functools.lru_cache(maxsize=None)
def _sinc_window(num_zeros, precision, beta, rolloff):
    from scipy.signal.windows import kaiser
    num_table = 2 ** precision
    n = num_table * num_zeros
    sinc_win = rolloff * np.sinc(rolloff * np.linspace(0, num_zeros, num=n + 1, endpoint=True))
    taper = kaiser(2 * n + 1, beta)[n:]
    win = taper * sinc_win
    win.flags.writeable = False
    return win, num_table


def filter_shape(orig_sr: int, res_type: str = "kaiser_best", sr: int = SR) -> Tuple[int, int, int]:
    """(nwin, num_table, index_step) of ``res_type`` at ``orig_sr -> sr``, from the table's parameters alone."""
    num_zeros, precision = RESAMPLE_FILTERS[res_type][:2]
    num_table = 2 ** precision
    return num_zeros * num_table + 1, num_table, int(min(1.0, float(sr) / orig_sr) * num_table)


@functools.lru_cache(maxsize=16)
def register_table(sample_ratio: float, n_out: int = REGISTER_HORIZON) -> np.ndarray:
    """resample_f's time register (``time_register += 1 / sample_ratio``, an fp64 running sum from 0.0) for outputs
    0 .. n_out - 1, in closed form per binade: int64 rows ``(t_b, base, k, e)`` with register(t) = (base + (t - t_b) k)
    2^e for t_b <= t < the next row's t_b, and a last row ``(n_out, 0, 0, 0)``.

    Within the binade [2^(e+52), 2^(e+53)) every sum is a multiple of the ulp 2^e and each step adds the increment
    rounded to that grid: a constant number of ulps, except that a tie may round the first step to the other parity
    (after it the register is even and stays so).  So the row starts where the next two steps agree and runs to the
    binade's end; a step that does not (the first, a parity fix, a step into the next binade) gets a one-output row and
    is taken by a real fp64 add.  A few rows per binade: O(log n_out) in all."""
    inc = 1.0 / sample_ratio
    rows, t, reg = [], 0, 0.0
    while t < n_out:
        if reg == 0.0:
            rows.append((t, 0, 0, 0))
            t, reg = t + 1, reg + inc
            continue
        e = math.frexp(reg)[1] - 53                    # reg in [2^(e+52), 2^(e+53)), ulp 2^e
        base = int(math.ldexp(reg, -e))
        r1 = reg + inc
        r2 = r1 + inc
        if r2 < math.ldexp(1.0, e + 53) and r2 - r1 == r1 - reg:
            k = int(math.ldexp(r1 - reg, -e))
            steps = min(-(-((1 << 53) - base) // k), n_out - t)          # outputs t .. t + steps - 1 in this binade
            rows.append((t, base, k, e))
            t, reg = t + steps, math.ldexp(float(base + (steps - 1) * k), e) + inc
        else:
            rows.append((t, base, 0, e))
            t, reg = t + 1, r1
    rows.append((n_out, 0, 0, 0))
    out = np.array(rows, dtype=np.int64)
    out.flags.writeable = False
    return out


def register_at(table: np.ndarray, t) -> np.ndarray:
    """The registers of outputs ``t`` (int array) from ``register_table`` rows, as the kernel evaluates them."""
    t = np.asarray(t, np.int64)
    r = np.searchsorted(table[:-1, 0], t, side="right") - 1
    return np.ldexp((table[r, 1] + (t - table[r, 0]) * table[r, 2]).astype(np.float64), table[r, 3].astype(np.int32))


def _frames(samples, channels: int) -> torch.Tensor:
    """``samples`` (numpy or torch; [n] or [n, channels]; fp32 or int16) as a tensor, refused with ``ValueError``
    otherwise.  Left on its device."""
    a = torch.as_tensor(samples)
    if a.dtype not in (torch.float32, torch.int16):
        raise ValueError(f"samples must be float32 or int16 (got {a.dtype})")
    if not (a.dim() == 1 and channels == 1) and not (a.dim() == 2 and a.shape[1] == channels):
        raise ValueError(f"samples must be [n] (mono) or [n, channels] with channels = {channels}, got shape {tuple(a.shape)}")
    return a


class Resampler(_lib.Handle):
    """``librosa.load``'s mono mix and resampling for audio decoded at ``orig_sr`` with ``channels`` (1 or 2) channels:
    ``resample(samples)`` returns what ``librosa.load(path, sr=16000)`` returns for those samples, as a CUDA fp32
    tensor.  The filter is resampy's ``res_type`` table (``resample_filter``), multiplied by the ratio when it is below
    one; its device copy is taken at construction.  Sample formats: float32 and PCM16 (decoded as s / 32768, as
    soundfile does), interleaved.  At ``orig_sr == 16000`` the mono mix is returned unchanged, as librosa does."""
    prefix, what = "lspa", "the resampler"

    def __init__(self, orig_sr: int, channels: int = 1, res_type: str = "kaiser_best", sr: int = SR,
                 device: Optional[torch.device] = None):
        if int(orig_sr) != orig_sr or orig_sr <= 0 or int(sr) != sr or sr <= 0:
            raise ValueError(f"sample rates must be positive integers (got {orig_sr}, {sr})")
        if channels not in (1, 2):
            raise ValueError(f"channels must be 1 or 2 (got {channels})")
        super().__init__(device)
        self.orig_sr, self.sr, self.channels, self.res_type = int(orig_sr), int(sr), int(channels), res_type
        self.sample_ratio = float(sr) / orig_sr
        self._create()
        if self.orig_sr == self.sr:
            return
        win, num_table = resample_filter(res_type)
        win = np.array(win, np.float64)
        if self.sample_ratio < 1:
            win *= self.sample_ratio
        delta = np.zeros_like(win)
        delta[:-1] = np.diff(win)
        self.nwin, self.num_table = win.shape[0], num_table
        self.index_step = int(min(1.0, self.sample_ratio) * num_table)
        self.wing = self.nwin // self.index_step     # the most taps of one wing
        self.call("load_resample_filter", win.ctypes.data, delta.ctypes.data, self.nwin, num_table, self.sample_ratio)
        self._reg = register_table(self.sample_ratio)

    def n_out(self, n_in: int) -> int:
        """``int(n_in * sample_ratio)``: the outputs resampy computes from ``n_in`` frames (it refuses fewer than one)."""
        return int(n_in * self.sample_ratio)

    def resample(self, samples) -> torch.Tensor:
        """CUDA fp32 ``[ceil(n * sample_ratio)]`` for ``n`` frames ([n] or [n, channels], numpy or torch, fp32 or int16).
        ``ValueError`` where resampy raises (fewer than one output).  Enqueued on the current stream; a host array goes
        through pinned memory, so there is no host synchronisation."""
        a = _frames(samples, self.channels)
        n = a.shape[0]
        if self.orig_sr == self.sr:
            return mono_mix(_lib.to_device(a, self.device, a.dtype))
        m = self.n_out(n)
        if m < 1:
            raise ValueError(f"input signal length={n} is too small to resample from {self.orig_sr}->{self.sr}")
        a = _lib.to_device(a, self.device, a.dtype)
        out = torch.empty(int(math.ceil(n * self.sample_ratio)), dtype=torch.float32, device=self.device)
        out[m:] = 0.0
        self._span(a, 0, 0, m, out)
        return out

    def _span(self, frames: torch.Tensor, first_in: int, first_out: int, n_out: int, out: torch.Tensor) -> None:
        fmt = 1 if frames.dtype == torch.int16 else 0
        with self.cuda_stream() as stream:
            self.call("resample_at", frames.data_ptr() if frames.numel() else None, fmt, self.channels, first_in,
                      frames.shape[0], first_out, n_out, self._reg.ctypes.data, self._reg.shape[0],
                      out.data_ptr() if n_out else None, stream)

    def stream(self) -> "ResampleStream":
        """A stream over one clip's native-rate frames: ``push(frames)`` returns the 16 kHz samples that became final,
        ``finish()`` the rest.  The concatenation equals ``resample`` of all the frames, bit for bit."""
        return ResampleStream(self)


def mono_mix(frames: torch.Tensor) -> torch.Tensor:
    """librosa's decoding and ``to_mono`` on device frames: fp32 s / 32768 for PCM16, then fp32 (c0 + c1) / 2."""
    x = frames.to(torch.float32) / 32768.0 if frames.dtype == torch.int16 else frames
    return x if x.dim() == 1 else (x[:, 0] + x[:, 1]) / 2.0


class ResampleStream:
    """``Resampler.resample`` over frames pushed in pieces.  Output t is returned by the push after which every input
    frame its right wing can read is in (``stream.resample_counts``): about ``nwin / index_step`` frames of latency,
    4 ms at 48 kHz with ``kaiser_best``.  ``finish()`` returns the outputs that read past the clip's end and the
    ``fix_length`` zero.  Only the frames from the left wing of the next output on are kept on the device."""

    def __init__(self, rs: Resampler):
        self._rs = rs
        self.frames = 0                         # frames pushed so far
        self.samples = 0                        # outputs returned so far
        self.finished = False
        self._tail = None                       # frames tail0 .. frames - 1
        self._tail0 = 0

    def push(self, frames) -> torch.Tensor:
        """[m] or [m, channels] frames (numpy or torch, fp32 or int16, one format per stream) -> the new 16 kHz samples."""
        if self.finished:
            raise RuntimeError("the stream has finished")
        a = _frames(frames, self._rs.channels)
        if self._tail is not None and a.dtype != self._tail.dtype:
            raise ValueError(f"one sample format per stream ({self._tail.dtype} so far, got {a.dtype})")
        a = _lib.to_device(a, self._rs.device, a.dtype)
        self.frames += a.shape[0]
        buf = torch.cat([self._tail, a]) if self._tail is not None and self._tail.numel() else a
        return self._emit(buf, False)

    def finish(self) -> torch.Tensor:
        """The rest, including ``fix_length``'s zero; ``ValueError`` where resampy would refuse the whole clip."""
        if self.finished:
            raise RuntimeError("the stream has finished")
        self.finished = True
        if self._rs.orig_sr != self._rs.sr and self._rs.n_out(self.frames) < 1:
            raise ValueError(f"input signal length={self.frames} is too small to resample from {self._rs.orig_sr}->"
                             f"{self._rs.sr}")
        buf = self._tail if self._tail is not None else torch.empty(0, dtype=torch.float32, device=self._rs.device)
        return self._emit(buf, True)

    def _emit(self, buf: torch.Tensor, finished: bool) -> torch.Tensor:
        from .stream import resample_counts
        rs = self._rs
        if rs.orig_sr == rs.sr:
            self.samples = self.frames
            self._tail = buf[:0]
            return mono_mix(buf)
        ready = resample_counts(self.frames, finished, rs.orig_sr, rs.res_type, rs.sr)
        computed = min(ready, rs.n_out(self.frames))          # beyond it: fix_length's zero
        out = torch.empty(ready - self.samples, dtype=torch.float32, device=rs.device)
        out[computed - self.samples:] = 0.0
        if computed > self.samples:
            rs._span(buf, self._tail0, self.samples, computed - self.samples, out)
        self.samples = ready
        if finished:
            self._tail = buf[:0]
            return out
        keep = int(register_at(rs._reg, ready)) - (rs.wing - 1)     # the left wing of the next output starts here
        keep = min(max(keep, self._tail0), self.frames)
        self._tail = buf[keep - self._tail0:].clone()
        self._tail0 = keep
        return out


def load_wav(path: str, sr: int = SR, res_type: str = "kaiser_best", device: Optional[torch.device] = None) -> torch.Tensor:
    """``librosa.load(path, sr=sr)`` for PCM16 and float32 WAV files with one or two channels, read with
    ``scipy.io.wavfile``: CUDA fp32 ``[ceil(n * sr / orig_sr)]``.  Other sample formats and more channels are refused
    with ``ValueError``."""
    from scipy.io import wavfile
    orig_sr, data = wavfile.read(path)
    if data.dtype not in (np.int16, np.float32):
        raise ValueError(f"{path}: {data.dtype} samples; only PCM16 and float32 WAV files are supported")
    if data.ndim > 2 or (data.ndim == 2 and data.shape[1] > 2):
        raise ValueError(f"{path}: {data.shape[1]} channels; at most two are supported")
    if data.ndim == 2 and data.shape[1] == 1:
        data = data[:, 0]
    return Resampler(orig_sr, 1 if data.ndim == 1 else 2, res_type, sr, device).resample(np.ascontiguousarray(data))


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
