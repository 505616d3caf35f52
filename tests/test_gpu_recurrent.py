"""The recurrent audio networks on the GPU (include/lspr.h): the APC encoder GRU stack and Audio2Mouth against the float64
truth of oracle/rnn_oracle.py.  Gate: max|kernel - truth| <= max(1e-5, 2 x the fp32 reference's own max error on the same
case) - for Audio2Mouth scaled by max(1, max|truth|) - and repeated runs bit-identical.  Also the golden fixtures, the
installed drop-ins and the device chain wav -> mel -> APC -> LLE -> mouth with no host synchronisation."""
import functools
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import rnn_oracle as R

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
GOLD_DIR = os.path.join(os.path.dirname(__file__), "golden", "rnn")


@functools.lru_cache(maxsize=None)
def _apc_sd(recipe, seed=0):
    return R.make_apc_state_dict(recipe, seed)


@functools.lru_cache(maxsize=None)
def _apc_case(recipe, T):
    """(mel, float64 truth, fp32 reference's max error) of one APC case."""
    sd = _apc_sd(recipe)
    mel = R.make_mel(T, seed=T)
    truth = R.apc_truth(sd, mel, device=DEV if T > 5000 else "cpu").cpu().numpy()
    ref_err = float(np.abs(R.apc_reference(sd, mel) - truth).max())
    return mel, truth, ref_err


@functools.lru_cache(maxsize=None)
def _encoder(recipe):
    from livespeechportraits_b200.recurrent import ApcEncoder
    return ApcEncoder(_apc_sd(recipe), device=DEV)


@pytest.mark.parametrize("cluster", [16, 8])
@pytest.mark.parametrize("T", [1, 2, 37, 1374, 72000])
@pytest.mark.parametrize("recipe", ["A", "B"])
def test_apc_against_truth(recipe, T, cluster):
    mel, truth, ref_err = _apc_case(recipe, T)
    enc = _encoder(recipe)
    x = torch.from_numpy(mel).to(DEV)
    got = enc.forward(x, cluster=cluster)
    again = enc.forward(x, cluster=cluster)
    assert got.shape == (T, 512) and got.dtype == torch.float32
    assert torch.equal(got, again)
    err = float(np.abs(got.cpu().numpy() - truth).max())
    gate = max(1e-5, 2 * ref_err)
    print(f"APC {recipe} T={T} cluster={cluster}: max|cuda - truth| {err:.3g}, fp32 reference {ref_err:.3g}, gate {gate:.3g}")
    assert err <= gate


def test_apc_cluster_variants_agree_and_residual():
    """Both cluster shapes sum every dot product in the same order, so they agree bit for bit; residual adds each
    512-wide layer's input except after the last layer."""
    sd = _apc_sd("B")
    mel = R.make_mel(200, seed=9)
    enc = _encoder("B")
    x = torch.from_numpy(mel).to(DEV)
    assert torch.equal(enc.forward(x, cluster=16), enc.forward(x, cluster=8))
    from livespeechportraits_b200.recurrent import ApcEncoder
    res = ApcEncoder(sd, device=DEV, residual=True).forward(x).cpu().numpy()
    truth = R.apc_truth(sd, mel, residual=True).numpy()
    ref_err = float(np.abs(R.apc_reference(sd, mel, residual=True) - truth).max())
    assert np.abs(res - truth).max() <= max(1e-5, 2 * ref_err)


@functools.lru_cache(maxsize=None)
def _mouth_case(recipe, n, ff):
    opt = R.default_mouth_opt(frame_future=ff)
    sd = R.make_mouth_state_dict(opt, recipe, seed=1)
    feats = R.make_feats(n, seed=n + ff)
    truth = R.mouth_truth(sd, feats, opt).numpy()
    ref_err = float(np.abs(R.generate_sequences(R.mouth_module(opt, sd), feats, opt) - truth).max())
    return opt, sd, feats, truth, ref_err


@pytest.mark.parametrize("ff", [0, 18])
@pytest.mark.parametrize("n", [2, 36, 1374])
@pytest.mark.parametrize("recipe", ["A", "B"])
def test_mouth_against_truth(recipe, n, ff):
    from livespeechportraits_b200.recurrent import MouthGenerator
    opt, sd, feats, truth, ref_err = _mouth_case(recipe, n, ff)
    gen = MouthGenerator(opt, sd, device=DEV)
    x = torch.from_numpy(feats).to(DEV)
    got = gen.generate(x)
    assert got.shape == (n // 2, 75) and torch.equal(got, gen.generate(x))
    err = float(np.abs(got.cpu().numpy() - truth).max())
    gate = max(1e-5, 2 * ref_err) * max(1.0, float(np.abs(truth).max()))
    print(f"mouth {recipe} n={n} ff={ff}: max|cuda - truth| {err:.3g}, fp32 reference {ref_err:.3g}, gate {gate:.3g}")
    assert err <= gate


def test_mouth_refusals():
    from livespeechportraits_b200.recurrent import MouthGenerator
    opt, sd, feats, _, _ = _mouth_case("A", 36, 18)
    gen = MouthGenerator(opt, sd, device=DEV)
    with pytest.raises(RuntimeError, match="is invalid for input of size"):
        gen.generate(torch.from_numpy(feats[:35]).to(DEV))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        gen.generate(torch.from_numpy(feats))
    with pytest.raises(NotImplementedError):
        MouthGenerator(R.default_mouth_opt(feature_decoder="WaveNet"), sd, device=DEV)


@pytest.mark.skipif(not os.path.isdir(GOLD_DIR), reason="no golden fixtures")
def test_goldens():
    """The fixtures written from the unmodified reference: the kernel against their float64 truth, gated by the reference's
    own recorded error."""
    from livespeechportraits_b200.recurrent import ApcEncoder, MouthGenerator
    names = sorted(f for f in os.listdir(GOLD_DIR) if f.endswith(".npz"))
    assert names
    for name in names:
        g = np.load(os.path.join(GOLD_DIR, name))
        rows = g["rows"]
        if str(g["kind"]) == "apc":
            sd = R.make_apc_state_dict(str(g["recipe"]), int(g["weight_seed"]))
            got = ApcEncoder(sd, device=DEV).forward(torch.from_numpy(R.make_mel(int(g["T"]), int(g["input_seed"]))).to(DEV))
            scale = 1.0
        else:
            opt = R.default_mouth_opt(frame_future=int(g["frame_future"]))
            sd = R.make_mouth_state_dict(opt, str(g["recipe"]), int(g["weight_seed"]))
            feats = R.make_feats(int(g["T"]), int(g["input_seed"]))
            got = MouthGenerator(opt, sd, device=DEV).generate(torch.from_numpy(feats).to(DEV))
            scale = max(1.0, float(np.abs(g["truth"]).max()))
        err = float(np.abs(got.cpu().numpy()[rows] - g["truth"]).max())
        gate = max(1e-5, 2 * float(g["ref_err"])) * scale
        print(f"{name}: max|cuda - truth| {err:.3g} on {len(rows)} rows, gate {gate:.3g}")
        assert err <= gate, name


def _stand_in_modules():
    """Modules named like the reference's, holding stand-ins for APC_encoder and Audio2FeatureModel."""
    net_mod = types.ModuleType("lspr_test_networks")
    a2f_mod = types.ModuleType("lspr_test_a2f_model")

    class APC_encoder(torch.nn.Module):
        def __init__(self, sd, residual):
            super().__init__()
            m = R.apc_module(sd)
            self.rnns = m.rnns
            self.rnn_residual = residual

        def forward(self, inputs, lengths):
            raise AssertionError("not installed")

    class Audio2FeatureModel:
        def __init__(self, opt, sd):
            self.Audio2Feature = R.mouth_module(opt, sd).to(DEV)
            self.device = DEV

        def generate_sequences(self, *a, **k):
            raise AssertionError("not installed")

    net_mod.APC_encoder = APC_encoder
    a2f_mod.Audio2FeatureModel = Audio2FeatureModel
    return net_mod, a2f_mod


def test_installed_drop_ins():
    from livespeechportraits_b200 import recurrent
    net_mod, a2f_mod = _stand_in_modules()
    sys.modules[net_mod.__name__] = net_mod
    sys.modules[a2f_mod.__name__] = a2f_mod
    try:
        recurrent.install(net_mod.__name__, a2f_mod.__name__)
        sd = _apc_sd("A")
        apc = net_mod.APC_encoder(sd, False).to(DEV).eval()
        mel, truth, ref_err = _apc_case("A", 37)
        x = torch.from_numpy(mel).to(DEV)[None]
        out = apc.forward(x, torch.Tensor([37]))
        assert out.is_cuda and out.shape == (1, 37, 512) and out.dtype == torch.float32
        assert np.abs(out[0].cpu().numpy() - truth).max() <= max(1e-5, 2 * ref_err)
        with pytest.raises(RuntimeError):
            apc.forward(x.cpu(), torch.Tensor([37]))
        with pytest.raises(ValueError):
            apc.forward(x, torch.Tensor([30]))
        with torch.no_grad():                                     # in-place weight change: the handle is re-packed
            apc.rnns[2].bias_hh_l0.add_(0.25)
        sd2 = {k: v.detach().cpu() for k, v in apc.state_dict().items()}
        t2 = R.apc_truth(sd2, mel).numpy()
        assert np.abs(apc.forward(x, torch.Tensor([37]))[0].cpu().numpy() - t2).max() <= max(1e-5, 2 * ref_err) * 4

        opt, msd, feats, mtruth, mref = _mouth_case("A", 36, 18)
        model = a2f_mod.Audio2FeatureModel(opt, msd)
        pred = model.generate_sequences(feats, 16000, 60, fill_zero=True, opt=opt)
        assert isinstance(pred, np.ndarray) and pred.dtype == np.float32 and pred.shape == (18, 75)
        assert np.abs(pred - mtruth).max() <= max(1e-5, 2 * mref) * max(1.0, float(np.abs(mtruth).max()))
        model.Audio2Feature.opt = R.default_mouth_opt(feature_decoder="WaveNet")
        with pytest.raises(NotImplementedError):
            model.generate_sequences(feats, 16000, 60, fill_zero=True, opt=opt)
    finally:
        sys.modules.pop(net_mod.__name__, None)
        sys.modules.pop(a2f_mod.__name__, None)


def test_device_chain_without_host_sync():
    """MelFrontEnd -> ApcEncoder -> ManifoldProjector -> MouthGenerator and HeadposeGenerator -> LandmarkPostprocessor, all on
    the device under torch's sync debug mode "error"; then the mouth track against MouthGenerator fed the oracle's APC
    features."""
    from livespeechportraits_b200.audio import MelFrontEnd
    from livespeechportraits_b200.headpose import HeadposeGenerator
    from livespeechportraits_b200.landmarks import Identity, LandmarkPostprocessor, StageParams
    from livespeechportraits_b200.manifold import ManifoldProjector
    from livespeechportraits_b200.recurrent import ApcEncoder, MouthGenerator
    from oracle import a2h_oracle as A
    from oracle import landmark_oracle as P
    from oracle import lle_oracle as L
    from oracle import mel_oracle as W
    a = W.make_audio(2 * 16000, 31)
    front = MelFrontEnd(W.make_basis(80), device=DEV)
    sd = _apc_sd("A")
    enc = ApcEncoder(sd, device=DEV)
    proj = ManifoldProjector(L.make_database(3000, 512, seed=32), device=DEV)
    mopt, msd = R.default_mouth_opt(), R.make_mouth_state_dict(R.default_mouth_opt(), "A", 3)
    mouth = MouthGenerator(mopt, msd, device=DEV)
    hopt = A.default_opt()
    head = HeadposeGenerator(hopt, A.make_state_dict(hopt, "B", 1), device=DEV)
    post = LandmarkPostprocessor(Identity(**P.make_identity(0)), device=DEV)
    prm = P.MAY
    x = torch.from_numpy(a).to(DEV)
    nframe = 120
    noise = torch.zeros((nframe, 12), device=DEV)
    pre = torch.zeros(12, device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        mel = front.logmel(x)
        feats = enc.forward(mel)
        blend = proj.project_features(feats, 10, 1.0)
        track = mouth.generate(blend)
        hfeats = torch.cat([blend, blend[-2 * hopt.frame_future:]]).reshape(-1, 1024)
        pose = head.generate(hfeats, pre, noise, 0.3)
        lm, sh = post.run(track, pose, StageParams(*(prm[k] for k in ("Feat_smooth_sigma", "AMP_method", "Feat_AMPs", "rot_AMP",
                                                                        "trans_AMP", "Head_smooth_sigma", "shoulder_AMP"))))
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert mel.shape == (240, 80) and feats.shape == (240, 512) and blend.shape == (240, 512)
    assert track.shape == (nframe, 75) and pose.shape == (nframe, 12) and lm.shape[:2] == (nframe, 73)
    feats_o = torch.from_numpy(R.apc_reference(sd, mel.cpu().numpy())).to(DEV)
    assert (feats - feats_o).abs().max().item() <= 1e-4
    track_o = mouth.generate(proj.project_features(feats_o, 10, 1.0))
    truth = R.mouth_truth(msd, proj.project_features(feats_o, 10, 1.0).cpu().numpy(), mopt).numpy()
    err = float((track - track_o).abs().max())
    print(f"chain: max|mouth(cuda APC) - mouth(oracle APC)| {err:.3g}, max|truth| {np.abs(truth).max():.3g}")
    assert err <= 1e-3 * max(1.0, float(np.abs(truth).max()))
