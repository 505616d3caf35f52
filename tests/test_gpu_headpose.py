"""Row N4 (SURVEY.md 8f) on the GPU: the persistent headpose kernel (include/lsph.h) against the oracle of the reference
loop (oracle/a2h_oracle.py), the golden vectors generated from the reference, and itself (cluster 8 vs single CTA).
Tolerance: 1e-4 max-abs on the GMM parameters and on the generated sequence (fp32 everywhere; only the summation order
differs from ATen's, and the error feeds back through the history)."""
import os

import numpy as np
import pytest
import torch

from oracle import a2h_oracle as A

pytestmark = pytest.mark.gpu
TOL = 1e-4
GOLD = os.path.join(os.path.dirname(__file__), "golden", "a2h_B_60.npz")


def _gen(opt, sd):
    from livespeechportraits_b200.headpose import HeadposeGenerator
    return HeadposeGenerator(opt, sd, device=torch.device("cuda", 0))


@pytest.mark.parametrize("recipe,cluster", [("A", 8), ("B", 8), ("B", 1)])
def test_generated_sequence_matches_the_oracle(recipe, cluster):
    opt = A.default_opt()
    sd = A.make_state_dict(opt, recipe, 3)
    audio = A.make_audio_feats(70, opt, 4)
    pre = np.linspace(-0.3, 0.2, 12).astype(np.float32)
    noise = A.reference_noise(55, 12, 1, seed=9)
    ref, rp = A.generate_sequences(sd, audio, pre, noise, opt, 0.3, return_params=True)
    g = _gen(opt, sd)
    pred, params = g.generate(audio, pre, noise, 0.3, return_params=True, cluster=cluster)
    pred, params = pred.cpu().numpy(), params.cpu().numpy()
    e1, e2 = np.abs(pred - ref).max(), np.abs(params - rp).max()
    print(f"headpose {recipe} cluster {cluster}: max|pred - oracle| = {e1:.3g}, max|params - oracle| = {e2:.3g} (|pred| up to {np.abs(ref).max():.2f})")
    assert e1 <= TOL and e2 <= TOL
    # Sample_GMM given the kernel's own parameters (losses.py:98-104): sample = noise * exp(-neg_log_sigma) * scale + mu
    samp = noise * (np.exp(-params[:, 13:25]) * np.float32(0.3)) + params[:, 1:13]
    assert np.abs(samp - pred).max() <= 1e-6
    # sigma_scale 0 (demo.py passes 0.3; 0 returns the means)
    p0, q0 = g.generate(audio, pre, noise, 0.0, return_params=True, cluster=cluster)
    assert torch.equal(p0, q0[:, 1:13])


def test_golden_vectors_from_the_reference_model():
    g = np.load(GOLD)
    opt = A.default_opt()
    sd = A.make_state_dict(opt, str(g["recipe"]), int(g["weight_seed"]))
    audio = A.make_audio_feats(int(g["n_audio"]), opt, int(g["audio_seed"]))
    gen = _gen(opt, sd)
    pred, params = gen.generate(audio, g["pre_headpose"], g["noise"], float(g["sigma_scale"]), return_params=True)
    assert np.abs(pred.cpu().numpy() - g["pred"]).max() <= TOL
    assert np.abs(params.cpu().numpy() - g["params"]).max() <= TOL


def test_full_clip_cluster_vs_single_cta_and_oracle_sample():
    """The 00083.wav clip length (687 audio rows -> 672 frames, SURVEY.md 8d): the 8-CTA cluster kernel and the single-CTA
    kernel agree over the whole clip, and the first 40 frames agree with the oracle."""
    opt = A.default_opt()
    sd = A.make_state_dict(opt, "B", 1)
    audio = A.make_audio_feats(687, opt, 2)
    pre = np.zeros(12, np.float32)                        # demo.py:211
    noise = A.reference_noise(672, 12, 1, seed=0)
    g = _gen(opt, sd)
    p8 = g.generate(audio, pre, noise, 0.3, cluster=8).cpu().numpy()
    p1 = g.generate(audio, pre, noise, 0.3, cluster=1).cpu().numpy()
    assert p8.shape == (672, 12) and np.isfinite(p8).all()
    assert np.abs(p8 - p1).max() <= TOL
    ref = A.generate_sequences(sd, audio[:55], pre, noise[:40], opt, 0.3)         # same first 40 frames: causal in the audio
    assert np.abs(p8[:40] - ref).max() <= TOL
    again = g.generate(audio, pre, noise, 0.3, cluster=8).cpu().numpy()
    assert np.array_equal(again, p8)                        # deterministic


def test_two_cuda_streams_share_one_generator():
    """Two different clips through one generator, enqueued on two CUDA streams with no synchronisation between the
    enqueues: every call owns its loop state and workspace, so each output equals its serial result bit for bit."""
    opt = A.default_opt()
    g = _gen(opt, A.make_state_dict(opt, "B", 1))
    dev = g.device
    clips = [(torch.from_numpy(A.make_audio_feats(n, opt, seed)).to(dev),
              torch.from_numpy(A.reference_noise(n - opt.frame_future, 12, 1, seed=seed)).to(dev))
             for n, seed in ((687, 2), (400, 5))]
    pre = torch.zeros(12, device=dev)
    serial = [g.generate(a, pre, nz, 0.3) for a, nz in clips]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(dev) for _ in clips]
    concurrent = []
    for s, (a, nz) in zip(streams, clips):
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):
            concurrent.append(g.generate(a, pre, nz, 0.3))
    torch.cuda.synchronize()
    assert all(torch.equal(c, r) for c, r in zip(concurrent, serial))


def test_drop_in_generate_sequences_keeps_signature_and_random_stream():
    import types
    from livespeechportraits_b200 import headpose
    opt = A.default_opt()
    sd = A.make_state_dict(opt, "B", 6)

    class FakeNet:                                           # stands where Audio2HeadposeModel.Audio2Headpose stands
        def state_dict(self):
            return sd
    model = types.SimpleNamespace(Audio2Headpose=FakeNet())
    audio = A.make_audio_feats(48, opt, 7)
    pre = np.zeros(12, np.float32)
    torch.manual_seed(21)
    out = headpose.generate_sequences(model, audio.reshape(-1), pre, fill_zero=True, sigma_scale=0.3, opt=opt)
    assert out.shape == (33, 12) and out.dtype == np.float64
    ref = A.generate_sequences(sd, audio, pre, A.reference_noise(33, 12, 1, seed=21), opt, 0.3)
    assert np.abs(out - ref).max() <= TOL
    assert headpose.generate_sequences(model, audio, pre, fill_zero=False, sigma_scale=0.3, opt=opt) is None
    # new weights in the SAME module object (load_state_dict copies in place): the cached device copy must follow
    sd2 = A.make_state_dict(opt, "B", 9)
    for k in sd:
        sd[k].copy_(sd2[k])
    torch.manual_seed(21)
    out2 = headpose.generate_sequences(model, audio.reshape(-1), pre, fill_zero=True, sigma_scale=0.3, opt=opt)
    ref2 = A.generate_sequences(sd2, audio, pre, A.reference_noise(33, 12, 1, seed=21), opt, 0.3)
    assert np.abs(out2 - ref2).max() <= TOL and np.abs(out2 - out).max() > 1e-3


def test_l2_loss_and_two_component_mixture():
    from livespeechportraits_b200.headpose import HeadposeGenerator
    opt = A.default_opt(loss="L2")
    sd = A.make_state_dict(opt, "B", 2)
    audio = A.make_audio_feats(40, opt, 3)
    pre = np.zeros(12, np.float32)
    g = HeadposeGenerator(opt, sd)
    pred, params = g.generate(audio, pre, None, 0.0, return_params=True)
    ref = A.generate_sequences(sd, audio, pre, np.zeros((25, 12), np.float32), opt, 0.0)
    assert params.shape == (25, 12) and np.abs(pred.cpu().numpy() - ref).max() <= TOL
    opt2 = A.default_opt(A2H_GMM_ncenter=2)
    sd2 = A.make_state_dict(opt2, "B", 2)
    g2 = HeadposeGenerator(opt2, sd2)
    noise = A.reference_noise(25, 12, 1, seed=1)
    uni = np.linspace(0.01, 0.99, 25).astype(np.float32)
    pred, params = g2.generate(audio, pre, noise, 0.3, uniform=uni, return_params=True)
    pred, params = pred.cpu().numpy(), params.cpu().numpy()
    assert params.shape == (25, 50)
    w = np.exp(params[:, :2] - params[:, :2].max(1, keepdims=True))
    w /= w.sum(1, keepdims=True)
    sel = (uni >= w[:, 0]).astype(int)                        # inverse CDF over the softmax weights
    mu = np.stack([params[i, 2 + sel[i] * 12: 2 + sel[i] * 12 + 12] for i in range(25)])
    nls = np.stack([params[i, 26 + sel[i] * 12: 26 + sel[i] * 12 + 12] for i in range(25)])
    assert np.abs(noise * (np.exp(-nls) * np.float32(0.3)) + mu - pred).max() <= 1e-5
