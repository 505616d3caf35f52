"""Row N6 (SURVEY.md 8f) on the GPU: the log-mel kernel of include/lspa.h against the float64 truth (a per-element bound
derived from the kernel's arithmetic, ``mel_oracle.error_bound``) and the fp32 restatement of the reference
(oracle/mel_oracle.py, 1e-5), the golden vectors generated from the reference, edge cases, determinism, the installed
drop-in, and the device chain mel -> APC GRU -> manifold projection."""
import functools
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import mel_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
GOLD_DIR = os.path.join(os.path.dirname(__file__), "golden", "mel")
GOLDENS = ["mel_00083_wav", "mel_synth_2s", "mel_synth_tail_randbasis", "mel_synth_one_frame", "mel_synth_empty",
           "mel_synth_L200", "mel_synth_L199", "mel_synth_L190_step67"]
TOL_ORACLE = 1e-5


@functools.lru_cache(maxsize=4)
def _front(basis_seed=None):
    from livespeechportraits_b200.audio import MelFrontEnd
    return MelFrontEnd(O.make_basis(80, basis_seed), device=DEV)


def _check(got, audio, basis, winlen=1 / 60, winstep=0.5 / 60, label="", windows=None):
    """Bound against the float64 truth and 1e-5 against the fp32 oracle; prints the worst ratios."""
    frame_len, step = int(16000 * winlen), 16000 * winstep
    assert got.dtype == np.float32 and got.shape == (O.n_windows(len(audio)), basis.shape[0])
    if windows is None:
        windows = np.arange(got.shape[0])
    t = O.logmel_truth(audio, basis, windows=windows, frame_len=frame_len, step=step)
    err = np.abs(got[windows].astype(np.float64) - t["out"])
    ratio = float((err / O.error_bound(t)).max()) if err.size else 0.0
    orc = O.compute_mel_one_sequence(audio, basis, winlen=winlen, winstep=winstep, batched=True)
    eo = float(np.abs(got - orc).max()) if got.size else 0.0
    print(f"{label}: {got.shape[0]} windows, max|cuda - truth| {err.max() if err.size else 0:.3g}, worst error/bound "
          f"{ratio:.3g}, max|cuda - fp32 oracle| {eo:.3g}")
    assert ratio <= 1.0 and eo <= TOL_ORACLE
    return eo


@pytest.mark.parametrize("name", GOLDENS)
def test_goldens_bound_and_oracle(name):
    g = np.load(os.path.join(GOLD_DIR, name + ".npz"))
    from livespeechportraits_b200.audio import MelFrontEnd
    front = MelFrontEnd(g["basis"], device=DEV)
    winlen, winstep = float(g["winlen"]), float(g["winstep"])
    got = front.logmel(g["audio"], winlen=winlen, winstep=winstep).cpu().numpy()
    assert got.shape == g["out"].shape
    if got.size:
        assert np.abs(got - g["out"]).max() <= TOL_ORACLE
    _check(got, g["audio"], g["basis"], winlen, winstep, name)


@pytest.mark.parametrize("frame_len", [190, 199, 200, 266])
@pytest.mark.parametrize("basis_seed", [None, 21])
def test_frame_lengths_and_bases(frame_len, basis_seed):
    a = O.make_audio(24000 + 37, 22)
    basis = O.make_basis(80, basis_seed)
    got = _front(basis_seed).logmel(a, winlen=frame_len / 16000).cpu().numpy()
    _check(got, a, basis, frame_len / 16000, 0.5 / 60, f"L={frame_len} basis={basis_seed}")


def test_other_mel_counts_and_no_normalisation():
    from livespeechportraits_b200.audio import MelFrontEnd
    a = O.make_audio(9000, 23)
    for n_mels in (1, 40, 128):
        basis = O.make_basis(n_mels, 24 + n_mels)
        got = MelFrontEnd(basis, device=DEV).logmel(a).cpu().numpy()
        _check(got, a, basis, label=f"n_mels={n_mels}")
    basis = O.make_basis(80)
    raw = _front().logmel(a, normalize=False).cpu().numpy()
    t = O.logmel_truth(a, basis, normalize=False)
    assert (np.abs(raw - t["out"]) <= O.error_bound(t, normalize=False)).all()


def test_short_clips_and_silence():
    f = _front()
    assert f.logmel(np.zeros(266, np.float32)).shape == (0, 80)          # shorter than one frame: empty
    assert f.logmel(np.zeros(0, np.float32)).shape == (0, 80)
    assert torch.equal(f.logmel(np.zeros(16000, np.float32)).cpu(), torch.zeros(120, 80))   # exactly 0.0
    for n in (267, 300, 533, 534, 800, 16000 + 133):                   # 2.. windows, the last ones short
        a = O.make_audio(n, n)
        _check(f.logmel(a).cpu().numpy(), a, O.make_basis(80), label=f"n={n}")


def test_float64_input_and_unaligned_device_pointer():
    f = _front()
    a64 = O.make_audio(20000, 25).astype(np.float64) * (1 + 2.0 ** -30)
    a32 = a64.astype(np.float32)
    ref = f.logmel(a32).cpu()
    assert torch.equal(f.logmel(a64).cpu(), ref)                         # float64 audio is its fp32 rounding
    assert torch.equal(f.logmel(torch.from_numpy(a64).to(DEV)).cpu(), ref)
    buf = torch.zeros(a32.shape[0] + 3, dtype=torch.float32, device=DEV)
    for off in (1, 2, 3):
        view = buf[off:off + a32.shape[0]]
        view.copy_(torch.from_numpy(a32))
        assert view.data_ptr() % 16 != 0
        assert torch.equal(f.logmel(view).cpu(), ref)


def test_runs_are_bit_identical():
    a = O.read_wav_fixture()
    f = _front()
    x = torch.from_numpy(a).to(DEV)
    first = f.logmel(x)
    for _ in range(3):
        assert torch.equal(f.logmel(x), first)


def test_ten_minute_clip():
    """72k windows: a wrong window start shows up as a large error against the truth somewhere along the clip."""
    a = O.make_audio(600 * 16000, 26)
    basis = O.make_basis(80)
    got = _front().logmel(a).cpu().numpy()
    assert got.shape == (72000, 80)
    windows = np.unique(np.concatenate([np.arange(0, 72000, 7), np.arange(71800, 72000)]))
    _check(got, a, basis, label="10 min", windows=windows)


def test_installed_drop_in_returns_the_reference_type():
    from livespeechportraits_b200 import audio as A
    mod = types.ModuleType("lspa_test_utils")
    mod.compute_mel_one_sequence = None
    sys.modules[mod.__name__] = mod
    try:
        A.install(mod.__name__)
        a = O.read_wav_fixture()
        out = mod.compute_mel_one_sequence(a, device="cuda")
        assert isinstance(out, np.ndarray) and out.dtype == np.float64 and out.shape == (1374, 80)
        assert np.array_equal(out, out.astype(np.float32))
        g = np.load(os.path.join(GOLD_DIR, "mel_00083_wav.npz"))
        assert np.abs(out - g["out"]).max() <= TOL_ORACLE
        out2 = mod.compute_mel_one_sequence(a.astype(np.float64), hop_length=1, fps=25, device="cpu")
        assert np.array_equal(out, out2)                                 # hop_length, fps and device change nothing
    finally:
        sys.modules.pop(mod.__name__, None)


def test_device_chain_mel_gru_manifold():
    """MelFrontEnd -> APC GRU (3 layers, 80 -> 512) -> ManifoldProjector on the device with no synchronising call, against
    the same chain fed the oracle's mel."""
    from livespeechportraits_b200.manifold import ManifoldProjector
    from oracle import lle_oracle as L
    a = O.make_audio(3 * 16000, 27)
    gru = O.ApcGru(seed=5).to(DEV).eval()
    db = L.make_database(4000, 512, seed=28)
    proj = ManifoldProjector(db, device=DEV)
    front = _front()
    x = torch.from_numpy(a).to(DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        mel = front.logmel(x)
        feats = gru(mel)
        blend = proj.project_features(feats, 10, 1.0)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert blend.is_cuda and blend.shape == (360, 512)
    mel_o = torch.from_numpy(O.compute_mel_one_sequence(a, O.make_basis(80)).astype(np.float32)).to(DEV)
    assert (mel - mel_o).abs().max().item() <= TOL_ORACLE
    feats_o = gru(mel_o)
    ef = (feats - feats_o).abs().max().item()
    blend_o = proj.project_features(feats_o, 10, 1.0)
    same = (proj.knn(feats, 10) == proj.knn(feats_o, 10)).all(1).float().mean().item()
    eb = (blend - blend_o).abs().max().item()
    print(f"chain: max|gru(cuda mel) - gru(oracle mel)| {ef:.3g}, neighbour rows equal {same:.3f}, max|blend diff| {eb:.3g}")
    assert ef <= 1e-4 and same >= 0.95
