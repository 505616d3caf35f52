"""librosa.load's resampling without a GPU: the register's closed form (``audio.register_table``) against the serial fp64
sum, the oracle restatement (oracle/resample_oracle.py) against analytic tones and its float64 truth, the mono mix
against numpy, the emission rule (``stream.resample_counts``) against brute force, and the argument checks of the new
``lspa_*`` entry points on a host-only handle."""
import contextlib
import ctypes as C

import numpy as np
import pytest

from livespeechportraits_b200 import _lib
from livespeechportraits_b200 import audio as A
from livespeechportraits_b200 import stream as S
from oracle import resample_oracle as R

RATES = [8000, 11025, 22050, 24000, 32000, 44100, 48000, 88200, 96000]


# ----------------------------------------------------------------------------------------------------------------------
# the time register
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("orig_sr", RATES)
def test_register_closed_form_is_the_serial_sum(orig_sr):
    ratio = 16000.0 / orig_sr
    n = 36_000_000                                       # 37.5 min at 16 kHz
    table = A.register_table(ratio)
    assert table.shape[0] <= 64 and table[-1, 0] == A.REGISTER_HORIZON
    got = A.register_at(table, np.arange(n))
    assert np.array_equal(got.view(np.int64), R.registers(n, ratio).view(np.int64))


def test_register_table_to_a_short_horizon():
    for orig_sr in RATES:
        ratio = 16000.0 / orig_sr
        for n in (1, 2, 3, 17, 1000):
            table = A.register_table(ratio, n)
            assert table[-1, 0] == n and np.all(np.diff(table[:, 0]) > 0)
            assert np.array_equal(A.register_at(table, np.arange(n)), R.registers(n, ratio))


# ----------------------------------------------------------------------------------------------------------------------
# the filters
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["kaiser_best", "kaiser_fast"])
def test_library_table_is_the_oracle_restatement(name):
    win, num_table = A.resample_filter(name)
    ref, ref_table = R.get_filter(name)
    assert num_table == ref_table == 512 and np.array_equal(win, ref)
    assert win.shape[0] == {"kaiser_best": 32769, "kaiser_fast": 8193}[name]
    assert A.filter_shape(48000, name)[:2] == (win.shape[0], num_table)
    assert A.filter_shape(48000, "kaiser_best")[2] == 170 and A.filter_shape(8000, "kaiser_best")[2] == 512
    assert win[0] == R.FILTERS[name][3]                  # the sinc's peak is the rolloff, the taper's 1
    with pytest.raises(ValueError, match="unknown filter"):
        A.resample_filter("polyphase")


# ----------------------------------------------------------------------------------------------------------------------
# known answer: tones well inside the pass band
# ----------------------------------------------------------------------------------------------------------------------
# Per case (input rate, tone, filter): the largest residual after fitting one gain, away from the clip ends.  Upsampling
# (8 kHz, index_step = num_table) is a true windowed-sinc interpolator: its residual is the stop-band level.  Downsampling
# truncates index_step = int(ratio * 512) (170 instead of 170.67 at 48 kHz): the taps sit slightly off the sinc's grid,
# the gain is 1.003 and the two wings are not mirror images, which leaves a residual of about 1.3e-4 of the amplitude at
# 440 Hz and 1.5e-3 at 5 kHz.  The bounds are about twice what the restatement reaches.
TONES = [(44100, 440, 2e-4), (44100, 5000, 2e-3), (48000, 440, 2e-4), (48000, 5000, 2e-3), (8000, 440, 1e-5),
         (8000, 2500, 1e-5)]


def _known_answer_failures():
    bad = []
    for orig_sr, f, tol in TONES:
        for name in ("kaiser_best", "kaiser_fast"):
            n = orig_sr // 2
            x = (0.5 * np.sin(2 * np.pi * f * np.arange(n) / orig_sr)).astype(np.float32)
            y, _ = R.resample_truth(x, orig_sr, name)
            t = R.registers(y.shape[0], 16000.0 / orig_sr)
            tone = 0.5 * np.sin(2 * np.pi * f * t / orig_sr)
            inner = slice(y.shape[0] // 8, y.shape[0] - y.shape[0] // 8)
            gain = np.dot(y[inner], tone[inner]) / np.dot(tone[inner], tone[inner])
            res = float(np.abs(y - gain * tone)[inner].max())
            if not (abs(gain - 1) <= 0.005 and res <= tol * (10 if name == "kaiser_fast" else 1)):
                bad.append((orig_sr, f, name, gain, res))
    return bad


def test_float64_truth_reproduces_tones():
    assert _known_answer_failures() == []


@contextlib.contextmanager
def _planted(defect):
    if defect == "window not scaled by the ratio":
        sf = R.scaled_filter
        patch = ("scaled_filter", lambda win, ratio: sf(win, 1.0))
    elif defect == "swapped wings":
        patch = ("wing_fracs", lambda frac, scale: (scale - frac, frac))
    else:
        wp = R.wing_params

        def patched(frac, num_table):
            offset, eta = wp(frac, num_table)
            return (offset, -eta) if defect == "sign of eta" else (offset + 1, eta)
        patch = ("wing_params", patched)
    old = getattr(R, patch[0])
    setattr(R, patch[0], patch[1])
    try:
        yield
    finally:
        setattr(R, patch[0], old)


@pytest.mark.parametrize("defect", ["window not scaled by the ratio", "swapped wings", "sign of eta",
                                    "off-by-one offset"])
def test_known_answer_catches_planted_defects(defect):
    with _planted(defect):
        assert _known_answer_failures() != []


# ----------------------------------------------------------------------------------------------------------------------
# restatement against its float64 truth
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("orig_sr", [8000, 11025, 44100, 48000, 96000])
@pytest.mark.parametrize("name", ["kaiser_best", "kaiser_fast"])
def test_restatement_within_its_bound_of_the_truth(orig_sr, name):
    rng = np.random.default_rng(orig_sr)
    n = orig_sr // 4 + 7
    frames = rng.integers(-32768, 32768, size=(n, 2)).astype(np.int16)
    y = R.resample(frames, orig_sr, name)
    truth, bound = R.resample_truth(frames, orig_sr, name)
    assert y.dtype == np.float32 and y.shape == (int(np.ceil(n * 16000 / orig_sr)),)
    assert np.all(np.abs(y - truth) <= bound)
    assert float((np.abs(y - truth) / np.maximum(bound, 1e-300)).max()) > 0.01      # the bound is not vacuous
    sub = np.array([0, 5, y.shape[0] // 2, y.shape[0] - 1])
    assert np.array_equal(R.resample(frames, orig_sr, name, outputs=sub), y[sub])


def test_fix_length_and_refusal():
    x = np.ones(44101, np.float32)                       # 44101 * 16000 / 44100 = 16000.36: one zero appended
    y = R.resample(x, 44100, "kaiser_fast")
    assert y.shape == (16001,) and y[-1] == 0.0 and y[-2] != 0.0
    assert R.resample(np.ones(3, np.float32), 48000).shape == (1,)
    with pytest.raises(ValueError, match="too small"):
        R.resample(np.ones(2, np.float32), 48000)


# ----------------------------------------------------------------------------------------------------------------------
# decoding and the mono mix
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float32, np.int16])
@pytest.mark.parametrize("channels", [1, 2])
def test_mono_mix_is_numpy_mean(dtype, channels):
    import torch
    rng = np.random.default_rng(channels)
    shape = (10007,) if channels == 1 else (10007, channels)
    if dtype == np.int16:
        frames = rng.integers(-32768, 32768, size=shape).astype(np.int16)
    else:
        frames = (rng.standard_normal(shape) * 10.0 ** rng.integers(-40, 3, size=shape)).astype(np.float32)
    y = R.decode(frames)
    want = np.mean(y.T, axis=0) if channels == 2 else y
    assert want.dtype == np.float32
    assert np.array_equal(R.to_mono(y), want)
    assert np.array_equal(A.mono_mix(torch.from_numpy(frames)).numpy(), want)


# ----------------------------------------------------------------------------------------------------------------------
# emission
# ----------------------------------------------------------------------------------------------------------------------
def _brute_counts(orig_sr, name, n_max):
    """Outputs ready after n = 0 .. n_max frames: the longest prefix t < int(n r) whose right wings (at most
    nwin // index_step frames past n(t)) are in; finished: ceil(n r), 0 where resampy refuses."""
    ratio = 16000.0 / orig_sr
    nwin, _, step = A.filter_shape(orig_sr, name)
    reach = R.registers(int(n_max * ratio) + 2, ratio).astype(np.int64) + nwin // step
    live, done = [], []
    for n in range(n_max + 1):
        total = int(n * ratio)
        live.append(int(np.sum(np.cumprod(reach[:total] <= n - 1))))
        done.append(int(np.ceil(n * ratio)) if total >= 1 else 0)
    return live, done


@pytest.mark.parametrize("orig_sr,name", [(48000, "kaiser_best"), (44100, "kaiser_best"), (8000, "kaiser_fast"),
                                          (11025, "kaiser_best"), (96000, "kaiser_fast")])
def test_resample_counts_match_brute_force(orig_sr, name):
    live, done = _brute_counts(orig_sr, name, 3000)
    assert orig_sr < 16000 or any(int(n * 16000 / orig_sr) != int(np.ceil(n * 16000 / orig_sr)) for n in range(3001))
    for n in range(3001):
        assert S.resample_counts(n, False, orig_sr, name) == live[n], n
        assert S.resample_counts(n, True, orig_sr, name) == done[n], n
    # far into a long clip, where the fp64 registers decide
    for n in (10 ** 8 + 1, 123456789, 2 ** 31 + 5):
        c = S.resample_counts(n, False, orig_sr, name)
        reg = A.register_table(16000.0 / orig_sr)
        reach = lambda t: int(A.register_at(reg, t)) + A.filter_shape(orig_sr, name)[0] // A.filter_shape(orig_sr, name)[2]
        assert reach(c - 1) <= n - 1 and (reach(c) > n - 1 or c == int(n * 16000 / orig_sr))
    assert S.resample_counts(12345, False, 16000) == S.resample_counts(12345, True, 16000) == 12345


def test_emitted_outputs_read_only_frames_that_are_in():
    """The exact reach of every emitted output (its right wing's length from its own offset) stays inside the frames."""
    for orig_sr, name in ((48000, "kaiser_best"), (44100, "kaiser_fast"), (8000, "kaiser_best")):
        ratio = 16000.0 / orig_sr
        nwin, num_table, step = A.filter_shape(orig_sr, name)
        reg = R.registers(5000, ratio)
        n = reg.astype(np.int64)
        offset = (((min(1.0, ratio) - min(1.0, ratio) * (reg - n)) * num_table).astype(np.int64))
        reach = n + (nwin - offset) // step
        for frames in range(0, 9000, 7):
            c = S.resample_counts(frames, False, orig_sr, name)
            assert np.all(reach[:c] <= frames - 1)


def test_counts_compose_with_portrait_counts():
    from livespeechportraits_b200.landmarks import StageParams
    from oracle import landmark_oracle as P
    prm = StageParams(*(P.MAY[k] for k in ("Feat_smooth_sigma", "AMP_method", "Feat_AMPs", "rot_AMP", "trans_AMP",
                                           "Head_smooth_sigma", "shoulder_AMP")))
    live, done = _brute_counts(48000, "kaiser_best", 48000 * 2)
    prev = 0
    for n in range(0, 48000 * 2 + 1, 97):
        got = S.portrait_counts(S.resample_counts(n, False, 48000), False, prm)
        assert got == S.portrait_counts(live[n], False, prm) and got >= prev
        assert S.ready_counts(S.resample_counts(n, False, 48000), False) == S.ready_counts(live[n], False)
        prev = got
    assert S.portrait_counts(S.resample_counts(96000, True, 48000), True, prm) == S.portrait_counts(done[96000], True, prm)


# ----------------------------------------------------------------------------------------------------------------------
# the C ABI on a host-only handle, and the Python refusals that need no device
# ----------------------------------------------------------------------------------------------------------------------
def test_host_only_handle_refuses_bad_arguments():
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.lspa_create(C.byref(h), -1) == 0
    try:
        win = np.ones(33, np.float64)
        assert lib.lspa_load_resample_filter(h, win.ctypes.data, win.ctypes.data, 33, 4, 0.5) == -2       # ENODEV
        for args, msg in (((None, win.ctypes.data, 33, 4, 0.5), b"null"), ((win.ctypes.data, win.ctypes.data, 1, 4, 0.5), b"nwin"),
                          ((win.ctypes.data, win.ctypes.data, 33, 0, 0.5), b"num_table"),
                          ((win.ctypes.data, win.ctypes.data, 33, 4, 0.0), b"sample_ratio"),
                          ((win.ctypes.data, win.ctypes.data, 33, 4, 0.1), b"must be >= 1")):
            assert lib.lspa_load_resample_filter(h, *args) == -1 and msg in lib.lspa_last_error(), args
        reg = np.ascontiguousarray(A.register_table(1 / 3, 1000))
        buf, out = C.c_void_p(16), C.c_void_p(16)                       # never dereferenced on a host-only handle

        def call(fmt=0, ch=2, first_in=0, n_in=10, first_out=0, n_out=3, table=reg, n_reg=None, frames=buf, dst=out):
            return lib.lspa_resample_at(h, frames, fmt, ch, first_in, n_in, first_out, n_out,
                                        table.ctypes.data if table is not None else None,
                                        table.shape[0] if n_reg is None else n_reg, dst, None)
        assert call() == -2 and b"host-only" in lib.lspa_last_error()
        assert call(fmt=1, ch=1) == -2
        bad = np.array(reg)
        bad[2, 0] = bad[1, 0]
        late = np.array(reg)
        late[0, 0] = 1
        for kw, msg in ((dict(fmt=2), b"format"), (dict(ch=3), b"channels"), (dict(ch=0), b"channels"),
                        (dict(n_in=-1), b">= 0"), (dict(n_out=-1), b">= 0"), (dict(first_in=-1), b">= 0"),
                        (dict(first_out=-2), b">= 0"), (dict(frames=None), b"null buffer"),
                        (dict(dst=None), b"null buffer"), (dict(table=None, n_reg=2), b"null buffer"),
                        (dict(n_reg=1), b"end row"), (dict(table=bad), b"increasing"), (dict(table=late), b"start at"),
                        (dict(first_out=998, n_out=3), b"table ends")):
            assert call(**kw) == -1 and msg in lib.lspa_last_error(), kw
        assert call(frames=None, n_in=0, dst=None, n_out=0) == -2         # empty spans need no buffers
    finally:
        lib.lspa_destroy(h)


def test_load_wav_refuses_other_formats(tmp_path):
    from scipy.io import wavfile
    for name, data in (("s32.wav", np.zeros((100, 2), np.int32)), ("f64.wav", np.zeros(100, np.float64)),
                       ("u8.wav", np.zeros(100, np.uint8)), ("three.wav", np.zeros((100, 3), np.int16))):
        wavfile.write(tmp_path / name, 48000, data)
        with pytest.raises(ValueError):
            A.load_wav(str(tmp_path / name))
