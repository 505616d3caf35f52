"""The oracle of the recurrent audio networks (oracle/rnn_oracle.py) and the weight packing of include/lspr.h, on the host:
the restatement against the fixtures written from the unmodified reference, the float64 truth against torch's own GRU /
LSTM in float64, the kernel's recurrence emulated on a host-only handle's packed arrays against the truth (gate order,
b_hn placement, BatchNorm fold, per-CTA W_hh slices, frame_future clamping), and the header against the binding."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from livespeechportraits_b200 import _lib
from livespeechportraits_b200.recurrent import ApcEncoder, MouthGenerator
from oracle import rnn_oracle as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD_DIR = os.path.join(ROOT, "tests", "golden", "rnn")
GOLDENS = sorted(f[:-4] for f in os.listdir(GOLD_DIR) if f.endswith(".npz"))


def test_golden_set_is_complete():
    apc = {f"apc_{r}_T{T}" for r in "AB" for T in (2, 37, 1374)}
    mouth = {f"mouth_{r}_n{n}_ff{ff}" for r in "AB" for n in (2, 36, 1374) for ff in (0, 18)}
    assert set(GOLDENS) == apc | mouth


@pytest.mark.parametrize("name", GOLDENS)
def test_restatement_and_truth_match_the_fixtures(name):
    g = np.load(os.path.join(GOLD_DIR, name + ".npz"))
    rows, T, ff = g["rows"], int(g["T"]), int(g["frame_future"])
    if str(g["kind"]) == "apc":
        sd = R.make_apc_state_dict(str(g["recipe"]), int(g["weight_seed"]))
        x = R.make_mel(T, int(g["input_seed"]))
        ref, truth = R.apc_reference(sd, x), R.apc_truth(sd, x).numpy()
    else:
        opt = R.default_mouth_opt(frame_future=ff)
        sd = R.make_mouth_state_dict(opt, str(g["recipe"]), int(g["weight_seed"]))
        x = R.make_feats(T, int(g["input_seed"]))
        ref, truth = R.generate_sequences(R.mouth_module(opt, sd), x, opt), R.mouth_truth(sd, x, opt).numpy()
    # the fixtures were written where the restatement was bit-equal to the reference; another CPU's BLAS may order fp32
    # sums differently, so the restatement is held to a few fp32 ulps here and the float64 truth to 1e-12
    assert np.abs(ref[rows] - g["ref"]).max() <= 2e-6
    assert np.abs(truth[rows] - g["truth"]).max() <= 1e-12
    assert abs(float(np.abs(ref - truth).max()) - float(g["ref_err"])) <= 2e-6


@pytest.mark.parametrize("recipe", ["A", "B"])
def test_truth_equals_torch_float64(recipe):
    sd = R.make_apc_state_dict(recipe, 2)
    mel = R.make_mel(37, 3)
    m = R.apc_module(sd).double()
    with torch.no_grad():
        y = torch.from_numpy(mel).double()[None]
        for rnn in m.rnns:
            y = rnn(y)[0]
    assert np.abs(y[0].numpy() - R.apc_truth(sd, mel).numpy()).max() <= 1e-12
    opt = R.default_mouth_opt()
    msd = R.make_mouth_state_dict(opt, recipe, 4)
    lstm = R.mouth_module(opt, msd).LSTM.double()
    x = torch.from_numpy(R.make_feats(40, 5)).double()
    with torch.no_grad():
        want = lstm(x[None])[0][0]
        got = x
        for k in range(3):
            p = lambda n: getattr(lstm, f"{n}_l{k}").detach()      # noqa: E731
            got = R.lstm_layer_truth(got, p("weight_ih"), p("weight_hh"), p("bias_ih"), p("bias_hh"))
    assert (want - got).abs().max().item() <= 1e-12


@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("recipe", ["A", "B"])
def test_apc_packing_emulated_equals_truth(recipe, residual):
    sd = R.exact_fold(R.make_apc_state_dict(recipe, 6))
    mel = R.make_mel(37, 7)
    enc = ApcEncoder(sd, device=-1, residual=residual)
    truth = R.apc_truth(sd, mel, residual=residual).numpy()
    for cl in (16, 8):
        assert np.abs(R.emulate_apc(enc.packed, mel, 3, residual, cl) - truth).max() <= 1e-12


@pytest.mark.parametrize("ff", [0, 18])
@pytest.mark.parametrize("recipe", ["A", "B"])
def test_mouth_packing_emulated_equals_truth(recipe, ff):
    opt = R.default_mouth_opt(frame_future=ff)
    sd = R.exact_fold(R.make_mouth_state_dict(opt, recipe, 8))
    feats = R.make_feats(36, 9)
    gen = MouthGenerator(opt, sd, device=-1)
    truth = R.mouth_truth(sd, feats, opt).numpy()
    assert np.abs(R.emulate_mouth(gen.packed, feats, ff) - truth).max() <= 1e-12


def test_batchnorm_fold_and_bias_fold_on_general_weights():
    opt = R.default_mouth_opt()
    sd = R.make_mouth_state_dict(opt, "B", 10)
    gen = MouthGenerator(opt, sd, device=-1)
    for s, (lin, bn) in ((0, ("downsample.0", "downsample.1")), (2, ("fc.0", "fc.1")), (3, ("fc.3", "fc.4"))):
        scale, shift = R.fold_bn_fp32(sd, lin, bn)
        assert np.array_equal(gen.packed(13 + 3 * s), scale) and np.array_equal(gen.packed(14 + 3 * s), shift)
    for s, lin in ((1, "downsample.3"), (4, "fc.6")):
        assert np.array_equal(gen.packed(12 + 3 * s), sd[lin + ".weight"].numpy().ravel())
        assert np.all(gen.packed(13 + 3 * s) == 1.0) and np.array_equal(gen.packed(14 + 3 * s), sd[lin + ".bias"].numpy())
    asd = R.make_apc_state_dict("B", 11)
    enc = ApcEncoder(asd, device=-1)
    bih, bhh = asd["rnns.1.bias_ih_l0"].numpy(), asd["rnns.1.bias_hh_l0"].numpy()
    b = enc.packed(4 + 1).reshape(512, 3)
    assert np.array_equal(b[:, 0], bih[:512] + bhh[:512]) and np.array_equal(b[:, 1], bih[512:1024] + bhh[512:1024])
    assert np.array_equal(b[:, 2], bih[1024:]) and np.array_equal(enc.packed(4 + 3), bhh[1024:])
    assert enc.packed(3).size == 512 and gen.packed(3).size == 0


def test_header_declares_exactly_the_bound_symbols():
    header = open(os.path.join(ROOT, "include", "lspr.h")).read()
    declared = set(re.findall(r"^(?:int|const char\*)\s+(lspr_\w+)\s*\(", header, flags=re.M))
    assert declared == set(_lib.SYMBOLS_R), declared ^ set(_lib.SYMBOLS_R)
    lib = _lib.load()
    for name in _lib.SYMBOLS_R:
        getattr(lib, name)


def test_host_only_handle_and_config_checks():
    lib = _lib.load()
    sd = R.make_apc_state_dict("A", 0)
    enc = ApcEncoder(sd, device=-1)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        enc.forward(torch.zeros(4, 80))
    assert lib.lspr_forward(enc._handle, None, 0, None, None, 0, 0, None) == -2          # LSPG_ENODEV: host-only handle
    assert "host-only" in (lib.lspr_last_error() or b"").decode()
    n = C.c_size_t()
    _lib.check_r(lib.lspr_workspace_bytes(enc._handle, 100, C.byref(n)))
    assert n.value == 4 * (100 * 1536 + 2 * 51200)
    bad = dict(sd)
    del bad["rnns.2.bias_hh_l0"]
    with pytest.raises(_lib.LspgError, match="missing parameter rnns.2.bias_hh_l0"):
        ApcEncoder(bad, device=-1)
    with pytest.raises(_lib.LspgError, match="hidden_size must be 512"):
        ApcEncoder(R.make_apc_state_dict("A", 0, hidden=256, layers=1), device=-1)
    prefixed = {"module." + k: v for k, v in sd.items()}
    prefixed["module.rnns.0.num_batches_tracked"] = torch.tensor(3)
    assert np.array_equal(ApcEncoder(prefixed, device=-1).packed(2), enc.packed(2))
    opt = R.default_mouth_opt(feature_decoder="WaveNet")
    with pytest.raises(NotImplementedError):
        MouthGenerator(opt, {}, device=-1)


def test_restatement_refuses_an_odd_row_count_like_the_reference():
    opt = R.default_mouth_opt()
    m = R.mouth_module(opt, R.make_mouth_state_dict(opt, "A", 0))
    with pytest.raises(RuntimeError, match="is invalid for input of size"):
        R.generate_sequences(m, R.make_feats(35, 1), opt)
