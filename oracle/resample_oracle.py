"""Restatement of ``librosa.load(path, sr=16000)`` after decoding: ``to_mono``, ``resampy.resample`` with a kaiser table
(``resample_f``) and ``fix_length``, as librosa 0.7.x and resampy 0.2.x publish them.  Neither library is installed
where this was written, so nothing here has been run against them; the restatement follows their source, numpy dtype
for numpy dtype:

- decoding (soundfile): PCM16 -> fp32 ``s / 32768``; float32 passes through.
- ``to_mono``: ``np.mean(y, axis=0)`` over the fp32 ``[C, n]`` view, i.e. fp32 ``(c0 + c1) / 2``.
- ``resample``: ``sample_ratio = float(sr_new) / sr_orig``, ``int(n * sample_ratio)`` outputs (below 1: ``ValueError``),
  the half window multiplied by ``sample_ratio`` when it is below one, ``interp_delta[:-1] = np.diff(interp_win)``, then
  ``resample_f`` (numba, no fastmath) into an fp32 ``y``: every tap is an fp64 weight ``win + eta * delta``, an fp64
  product with the sample and an fp64 sum with ``y``, rounded to fp32 on the store.
- ``fix_length``: zero-pad to ``int(np.ceil(n * sample_ratio))``.

``resample_f`` is vectorised over outputs and loops over tap index in reference order, with per-output masks for the
wing lengths; its register is ``np.add.accumulate``, the serial fp64 sum itself.  ``outputs`` selects output indices, so
long clips can be checked at chosen windows.  ``resample_truth`` takes the same taps in fp64 and returns a per-element
bound on the restatement's distance from it.
"""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np

# resampy's shipped tables: num_zeros, precision, Kaiser beta, rolloff
FILTERS = {"kaiser_best": (64, 9, 14.769656459379492, 0.9475937167399596),
           "kaiser_fast": (16, 9, 8.555504641634386, 0.85)}


def sinc_window(num_zeros: int = 64, precision: int = 9, window=None, rolloff: float = 0.945) -> Tuple[np.ndarray, int]:
    """resampy.filters.sinc_window: the right half of a windowed sinc, ``2**precision`` entries per zero crossing."""
    num_bits = 2 ** precision
    n = num_bits * num_zeros
    sinc_win = rolloff * np.sinc(rolloff * np.linspace(0, num_zeros, num=n + 1, endpoint=True))
    taper = window(2 * n + 1)[n:]
    return taper * sinc_win, num_bits


def get_filter(name: str) -> Tuple[np.ndarray, int]:
    """The kaiser table ``name`` as resampy builds it (its ``.npz`` may differ in the last bits)."""
    from scipy.signal.windows import kaiser
    num_zeros, precision, beta, rolloff = FILTERS[name]
    return sinc_window(num_zeros, precision, lambda m: kaiser(m, beta), rolloff)


def decode(frames: np.ndarray) -> np.ndarray:
    """soundfile's float32 view of PCM16 or float32 frames ``[n]`` / ``[n, C]``."""
    if frames.dtype == np.int16:
        return frames.astype(np.float32) / np.float32(32768)
    assert frames.dtype == np.float32
    return frames


def to_mono(y: np.ndarray) -> np.ndarray:
    """librosa's ``to_mono`` on decoded frames ``[n]`` / ``[n, 2]``, spelled out: fp32 ``(c0 + c1) / 2``."""
    if y.ndim == 1:
        return y
    return (y[:, 0] + y[:, 1]) / np.float32(2)


def scaled_filter(win: np.ndarray, sample_ratio: float) -> Tuple[np.ndarray, np.ndarray]:
    """``interp_win`` (times ``sample_ratio`` below one) and ``interp_delta`` as resampy hands them to resample_f."""
    win = np.array(win, np.float64)
    if sample_ratio < 1:
        win *= sample_ratio
    delta = np.zeros_like(win)
    delta[:-1] = np.diff(win)
    return win, delta


def registers(n_out: int, sample_ratio: float) -> np.ndarray:
    """resample_f's ``time_register`` at outputs 0 .. n_out - 1: the serial fp64 sum 0 + 1/r + 1/r + ..."""
    reg = np.zeros(n_out, np.float64)
    if n_out > 1:
        np.add.accumulate(np.full(n_out - 1, 1.0 / sample_ratio), out=reg[1:])
    return reg


def wing_fracs(frac: np.ndarray, scale: float) -> Tuple[np.ndarray, np.ndarray]:
    """The filter phase of the left wing and of the right wing (``scale - frac``)."""
    return frac, scale - frac


def wing_params(frac: np.ndarray, num_table: int) -> Tuple[np.ndarray, np.ndarray]:
    """``offset = int(frac * num_table)`` and ``eta``, its fractional part."""
    index_frac = frac * num_table
    offset = index_frac.astype(np.int64)
    return offset, index_frac - offset


def _taps(x: np.ndarray, sample_ratio: float, win: np.ndarray, delta: np.ndarray, num_table: int, t: np.ndarray,
          reg: np.ndarray):
    """Yields, for each tap in reference order (left wing i = 0, 1, ..., then right wing k = 0, 1, ...), the fp64
    product ``weight * x`` of every selected output, 0 where the output has no such tap."""
    scale = min(1.0, sample_ratio)
    index_step = int(scale * num_table)
    nwin, n_orig = win.shape[0], x.shape[0]
    r = reg[t]
    n = r.astype(np.int64)
    fl, fr = wing_fracs(scale * (r - n), scale)
    for side, frac in (("left", fl), ("right", fr)):
        offset, eta = wing_params(frac, num_table)
        count = (nwin - offset) // index_step
        count = np.minimum(n + 1, count) if side == "left" else np.minimum(n_orig - n - 1, count)
        for i in range(int(count.max()) if count.size else 0):
            live = i < count
            j = np.where(live, offset + i * index_step, 0)
            weight = win[j] + eta * delta[j]
            src = np.where(live, n - i if side == "left" else n + i + 1, 0)
            yield np.where(live, weight * x[src].astype(np.float64), 0.0), live


def _prepare(frames: np.ndarray, orig_sr: int, name: str, sr: int, outputs: Optional[np.ndarray]):
    x = to_mono(decode(frames))
    sample_ratio = float(sr) / orig_sr
    n_out = int(x.shape[0] * sample_ratio)
    if n_out < 1:
        raise ValueError(f"Input signal length={x.shape[0]} is too small to resample from {orig_sr}->{sr}")
    table, num_table = get_filter(name)
    win, delta = scaled_filter(table, sample_ratio)
    total = int(np.ceil(x.shape[0] * sample_ratio))
    t = np.arange(total) if outputs is None else np.asarray(outputs, np.int64)
    inside = t < n_out                                   # the rest is fix_length's zero
    reg = registers(int(t[inside].max()) + 1 if inside.any() else 0, sample_ratio)
    return x, sample_ratio, win, delta, num_table, t, inside, reg, total


def resample(frames: np.ndarray, orig_sr: int, name: str = "kaiser_best", sr: int = 16000,
             outputs: Optional[np.ndarray] = None) -> np.ndarray:
    """``librosa.load``'s samples for decoded ``frames`` (int16 or float32, ``[n]`` or ``[n, 2]``) at ``orig_sr``: fp32
    ``[ceil(n * sr / orig_sr)]``, or the outputs at the indices ``outputs``."""
    if orig_sr == sr:
        y = to_mono(decode(frames))
        return y if outputs is None else y[outputs]
    x, ratio, win, delta, num_table, t, inside, reg, _ = _prepare(frames, orig_sr, name, sr, outputs)
    y = np.zeros(t.shape[0], np.float32)
    ti = t[inside]
    yi = np.zeros(ti.shape[0], np.float32)
    for p, _ in _taps(x, ratio, win, delta, num_table, ti, reg):
        yi = (yi.astype(np.float64) + p).astype(np.float32)
    y[inside] = yi
    return y


def resample_truth(frames: np.ndarray, orig_sr: int, name: str = "kaiser_best", sr: int = 16000,
                   outputs: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray]:
    """The same taps as ``resample``, summed in fp64 (``S``), and a bound ``B`` with ``|resample - S| <= B``.

    Derivation.  Let the products of one output be p_0, p_1, ... (fp64, identical in both: the weights and products
    are computed the same way).  The truth takes S_{j+1} = (S_j + p_j)(1 + e_j), |e_j| <= v = 2^-53; the restatement
    y_{j+1} = (y_j + p_j)(1 + d_j), |d_j| <= u = 2^-24, or y_j + p_j plus an absolute error of at most 2^-150 when the
    result is subnormal in fp32.  With E_j = y_j - S_j:
        E_{j+1} = E_j (1 + d_j) + (S_j + p_j)(d_j - e_j)   (+ the subnormal term),
    and |S_j + p_j| <= |S_{j+1}| (1 + 2v), so
        |E_{j+1}| <= |E_j| (1 + u) + |S_{j+1}| (u + v)(1 + 2v) + 2^-150.
    ``B`` is that recurrence from E_0 = 0, evaluated in fp64 and widened by 1e-12 relative for its own roundings.
    The fix_length zeros are exact (B = 0)."""
    u, v = 2.0 ** -24, 2.0 ** -53
    if orig_sr == sr:
        y = resample(frames, orig_sr, name, sr, outputs).astype(np.float64)
        return y, np.zeros_like(y)
    x, ratio, win, delta, num_table, t, inside, reg, _ = _prepare(frames, orig_sr, name, sr, outputs)
    s = np.zeros(int(inside.sum()), np.float64)
    b = np.zeros_like(s)
    for p, live in _taps(x, ratio, win, delta, num_table, t[inside], reg):
        s = s + p
        b = np.where(live, b * (1 + u) + np.abs(s) * (u + v) * (1 + 2 * v) + 2.0 ** -150, b)
    truth, bound = np.zeros(t.shape[0]), np.zeros(t.shape[0])
    truth[inside], bound[inside] = s, b * (1 + 1e-12)
    return truth, bound
