"""Row N6 (SURVEY.md 8f), CPU part: the oracle of the log-mel front end (oracle/mel_oracle.py) pinned against the golden
vectors generated from the reference's compute_mel_one_sequence / Audio2Mel and, where the reference checkout exists,
against those functions themselves; the fp32 normalisation; the window starts; the Slaney filterbank's structure; the C
ABI's argument checking on a host-only handle; the drop-in's refusals and install() on a stand-in funcs.utils module."""
import ctypes as C
import inspect
import math
import os
import sys
import types

import numpy as np
import pytest
import torch

from livespeechportraits_b200 import _lib, audio
from oracle import mel_oracle as O

GOLD_DIR = os.path.join(os.path.dirname(__file__), "golden", "mel")
GOLDENS = ["mel_00083_wav", "mel_synth_2s", "mel_synth_tail_randbasis", "mel_synth_one_frame", "mel_synth_empty",
           "mel_synth_L200", "mel_synth_L199", "mel_synth_L190_step67"]


def _golden(name):
    return np.load(os.path.join(GOLD_DIR, name + ".npz"))


@pytest.mark.parametrize("name", GOLDENS)
def test_restatement_matches_the_goldens_bit_for_bit(name):
    """Written by oracle/make_golden_mel.py from the UNMODIFIED reference, where the restatement was bit-equal to it."""
    g = _golden(name)
    got = O.compute_mel_one_sequence(g["audio"], g["basis"], winlen=float(g["winlen"]), winstep=float(g["winstep"]))
    assert got.dtype == np.float64 and got.shape == (O.n_windows(len(g["audio"])), 80)
    assert np.array_equal(got, g["out"].astype(np.float64))


@pytest.mark.parametrize("name", ["mel_00083_wav", "mel_synth_2s", "mel_synth_L190_step67"])
def test_float64_truth_vs_the_reference_within_recorded_error(name):
    g = _golden(name)
    frame_len, step = int(16000 * float(g["winlen"])), 16000 * float(g["winstep"])
    t = O.logmel_truth(g["audio"], g["basis"], frame_len=frame_len, step=step)
    err = np.abs(g["out"] - t["out"])
    assert err.max() <= float(g["err_truth"]) + 1e-12 and float(g["err_truth"]) <= 1e-5
    assert (err <= O.error_bound(t)).all()          # the fp32 reference meets the kernel's bound too


@pytest.mark.skipif(not O.reference_available(), reason="reference checkout not present on this machine")
def test_restatement_is_bit_equal_to_the_live_reference():
    basis = O.make_basis(80, 11)
    ref = O.reference_functions(basis)["compute_mel_one_sequence"]
    for n, winlen, winstep in ((5000, 1 / 60, 0.5 / 60), (4000, 195 / 16000, 0.4 / 60)):
        a = O.make_audio(n, 12)
        assert np.array_equal(ref(a, winlen=winlen, winstep=winstep),
                              O.compute_mel_one_sequence(a, basis, winlen=winlen, winstep=winstep))
    a64 = O.make_audio(3000, 13).astype(np.float64) * (1 + 2.0 ** -40)    # float64 audio: rounded to fp32 per clip
    assert np.array_equal(ref(a64), O.compute_mel_one_sequence(a64, basis))
    assert np.array_equal(ref(a64), O.compute_mel_one_sequence(a64.astype(np.float32), basis))


def test_normalisation_is_the_fp32_formula_on_a_dense_sweep():
    """(x - m) / -m evaluated by torch on fp32 equals normalize_fp32 everywhere on a dense sweep of the log range; the
    float64 evaluation rounded once does not."""
    x = np.concatenate([np.linspace(-11.6, 6.0, 2_000_001, dtype=np.float32),
                        np.random.default_rng(0).uniform(-11.6, 6.0, 1_000_000).astype(np.float32),
                        np.float32([math.log(1e-5), np.log(np.float32(1e-5)), 0.0, -0.0])])
    got = ((torch.from_numpy(x) - O.MIN_MEL) / -O.MIN_MEL).numpy()
    assert np.array_equal(got, O.normalize_fp32(x))
    f64 = ((x.astype(np.float64) - O.MIN_MEL) / -O.MIN_MEL).astype(np.float32)
    assert not np.array_equal(got, f64)
    # a silent window: log(clamp(0, 1e-5)) normalises to exactly 0.0
    silent = torch.log(torch.clamp(torch.zeros(1), min=1e-5))
    assert ((silent - O.MIN_MEL) / -O.MIN_MEL).item() == 0.0


def test_window_starts_are_the_truncated_fp64_products():
    step = 16000 * (0.5 / 60)
    assert step == 133.33333333333334
    n = 2_000_000
    st = O.window_starts(n, step)
    i = np.arange(n)
    assert np.array_equal(st, (400 * i) // 3)
    assert np.array_equal(st, np.trunc(i * step).astype(np.int64))
    for s in (66.66666666666667, 133.0, 100.5, 0.0):
        assert np.array_equal(O.window_starts(5000, s), [int(k * s) for k in range(5000)])
    assert O.n_windows(183296) == 1374 and O.n_windows(266) == 0 and O.n_windows(267) == 2


def test_frame_lengths_outside_190_to_266_raise_before_any_device_work():
    for winlen in (189 / 16000, 100 / 16000, 267 / 16000, 1 / 30):
        with pytest.raises(ValueError, match="frame length"):
            audio.compute_mel_one_sequence(np.zeros(20000, np.float32), winlen=winlen)
    # the reference itself fails there: the reflect pad needs p < L, and the row assignment needs one stft frame
    with pytest.raises(RuntimeError):
        O.audio2mel(torch.zeros(1, 1, 189), torch.zeros(80, 257))
    assert O.audio2mel(torch.zeros(1, 1, 267), torch.zeros(80, 257)).shape == (1, 80, 2)
    for L in (189, 267):
        if O.reference_available():
            with pytest.raises(Exception):
                O.reference_functions(np.zeros((80, 257), np.float32))["compute_mel_one_sequence"](
                    np.zeros(2000, np.float32), winlen=L / 16000)
    for L in (190, 266):
        assert O.audio2mel(torch.zeros(1, 1, L), torch.zeros(80, 257)).shape == (1, 80, 1)


def test_slaney_filterbank_structure():
    sr, n_fft, n_mels, fmin, fmax = 16000, 512, 80, 90.0, 7600.0
    B = O.slaney_mel(sr, n_fft, n_mels, fmin, fmax)
    assert B.dtype == np.float32 and B.shape == (80, 257) and (B >= 0).all()
    edges = O.mel_band_edges(sr, n_mels, fmin, fmax)
    assert edges[0] == pytest.approx(fmin, rel=1e-12) and edges[-1] == pytest.approx(fmax, rel=1e-12)
    # the edges are equally spaced on the Slaney scale: linear below 1 kHz, logarithmic above
    mel = np.where(edges < 1000, edges * 3 / 200, 15 + np.log(edges / 1000) * 27 / np.log(6.4))
    assert np.allclose(np.diff(mel), np.diff(mel)[0], rtol=1e-9)
    f = np.arange(257) * sr / n_fft
    for i in range(n_mels):
        lo, c, hi = edges[i], edges[i + 1], edges[i + 2]
        peak = 2.0 / (hi - lo)                         # area normalisation: the triangle's height
        tri = np.maximum(0, np.minimum((f - lo) / (c - lo), (hi - f) / (hi - c))) * peak
        assert np.allclose(B[i], tri, rtol=1e-5, atol=1e-9), i
        assert (B[i][(f <= lo) | (f >= hi)] == 0).all()
        assert B[i].max() <= peak * (1 + 1e-6)
    assert (B[:, (f < fmin) | (f > fmax)] == 0).all()
    assert np.array_equal(audio.mel_basis(), B) or _has_librosa()


def _has_librosa():
    try:
        import librosa  # noqa: F401
        return True
    except ImportError:
        return False


def test_test_audio_is_deterministic_and_covers_its_cases():
    a = O.make_audio(12000 * 2, 3)
    assert a.dtype == np.float32 and np.array_equal(a, O.make_audio(12000 * 2, 3)) and np.abs(a).max() <= 1.0
    assert (a[4000:6000] == 0).all()                                     # silence
    assert (np.abs(a[6000:8000]) == 1.0).sum() > 100                     # clipped at exactly +-1
    assert not np.array_equal(a, O.make_audio(12000 * 2, 4))


def test_host_only_handle_argument_checks():
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.lspa_create(None, -1) == -1
    assert lib.lspa_create(C.byref(h), -2) == -1
    if not torch.cuda.is_available():
        assert lib.lspa_create(C.byref(h), 0) == -2                       # no device, no fallback
    assert lib.lspa_create(C.byref(h), -1) == 0
    try:
        basis = np.zeros((129, 257), np.float32)
        load = lambda n_mels, n_bins, p=basis.ctypes.data: lib.lspa_load_mel_basis(h, p, n_mels, n_bins)   # noqa: E731
        for n_mels, n_bins in ((0, 257), (-1, 257), (129, 257), (80, 256), (80, 258), (80, 0)):
            assert load(n_mels, n_bins) == -1, (n_mels, n_bins)
        assert load(80, 257, None) == -1
        assert load(80, 257) == -2 and b"no CPU path" in lib.lspa_last_error()
        assert load(1, 257) == -2 and load(128, 257) == -2
        buf = (C.c_float * 16)()
        p = C.cast(buf, C.c_void_p)
        mel = lambda a, n, nw, L, step=133.33333333333334, out=p: lib.lspa_logmel_at(h, a, 0, n, 0, nw, L, step, 1, out, None)   # noqa: E731
        for L in (189, 267, 0, -5, 512):
            assert mel(p, 20000, 10, L) == -1, L
        assert b"frame_len" in lib.lspa_last_error()
        assert mel(p, 20000, -1, 266) == -1
        assert mel(p, -1, 10, 266) == -1
        for step in (-1.0, float("nan"), float("inf"), 1e300):
            assert mel(p, 20000, 10, 266, step) == -1, step
        assert mel(None, 20000, 10, 266) == -1
        assert mel(p, 20000, 10, 266, out=None) == -1
        for L in (190, 199, 200, 266):
            assert mel(p, 20000, 10, L) == -2 and b"no CPU path" in lib.lspa_last_error()
        assert mel(None, 0, 0, 266, out=None) == -2                        # an empty clip is valid
        assert mel(p, 20000, (1 << 31) - 1, 266, 133.0) == -2
    finally:
        assert lib.lspa_destroy(h) == 0
    assert lib.lspa_destroy(None) == 0


def test_python_layer_refuses_the_cpu():
    with pytest.raises(RuntimeError, match="no CPU path"):
        audio.MelFrontEnd(device=torch.device("cpu"))


def test_install_replaces_the_function_with_the_reference_signature():
    mod = types.ModuleType("lspa_stand_in_utils")
    mod.compute_mel_one_sequence = O.compute_mel_one_sequence
    sys.modules[mod.__name__] = mod
    try:
        audio.install(mod.__name__)
        assert mod.compute_mel_one_sequence is audio.compute_mel_one_sequence
        sig = str(inspect.signature(mod.compute_mel_one_sequence))
        assert sig == ("(audio, hop_length=133, winlen=0.016666666666666666, winstep=0.008333333333333333, sr=16000, "
                       "fps=60, device='cpu')"), sig
        if O.reference_available():
            ref = O.reference_functions(np.zeros((80, 257), np.float32))["compute_mel_one_sequence"]
            assert inspect.signature(ref) == inspect.signature(mod.compute_mel_one_sequence)
        if not torch.cuda.is_available():
            with pytest.raises(RuntimeError, match="no CPU path"):
                mod.compute_mel_one_sequence(np.zeros(2000, np.float32))
    finally:
        sys.modules.pop(mod.__name__, None)
