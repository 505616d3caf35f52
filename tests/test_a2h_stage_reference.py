"""The float64 stage truths of the Audio2Headpose loop (tests/a2h_stage_reference.py) on the CPU: they compose to the
float64 incremental emulator, the fp32 host emulator stays within every bound when read back span by span exactly as
tests/test_gpu_headpose_stages.py reads the kernel, each planted defect in that emulator is caught, and the state and
workspace layouts the GPU test reads are pinned on a host-only handle."""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import a2h_incremental as INC  # noqa: E402
import a2h_stage_reference as SR  # noqa: E402
from oracle import a2h_oracle as A  # noqa: E402

# (name, option overrides, frames): the configurations lsph_create accepts beyond the shipped one that a CPU can run
CONFIGS = [
    ("default", {}, 6),
    ("8x2", dict(A2H_wavenet_residual_layers=8), 3),
    ("1x16", dict(A2H_wavenet_residual_layers=1, A2H_wavenet_residual_blocks=16), 6),
    ("ncenter5", dict(A2H_GMM_ncenter=5), 6),
    ("L2", dict(loss="L2"), 6),
    ("no_bias", dict(A2H_wavenet_use_bias=False), 6),
    ("ff0", dict(frame_future=0), 6),
]


def _clip(opt, nframe, seed=4):
    audio = A.make_audio_feats(nframe + opt.frame_future, opt, seed)
    pre = np.linspace(-0.3, 0.2, opt.A2H_wavenet_input_channels).astype(np.float32)
    noise = A.reference_noise(nframe, opt.A2H_GMM_ndim, 1, seed=9)
    uniform = np.linspace(0.03, 0.97, nframe).astype(np.float32) if opt.A2H_GMM_ncenter > 1 else None
    return audio, pre, noise, uniform


def run_emulator(net, audio, pre, noise, uniform, sigma, defect=None, label=""):
    """The emulator driven span by span like the kernel in the GPU test, every span checked.  Returns (gate, params)."""
    nframe = audio.shape[0] - net.ff
    state = np.zeros(net.state_floats(), np.float32)
    gate = SR.Gate(label)
    preds, params = [], []
    for f0, n in SR.span_plan(net, nframe):
        lo, hi = SR.span_rows(net, f0, n)
        nz = noise[f0:f0 + n] if noise is not None else None
        un = uniform[f0:f0 + n] if uniform is not None else None
        p, q, ws = SR.emulate_span(net, audio[lo:hi], lo, f0, n, pre, nz, un, sigma, state, defect)
        preds.append(p)
        params.append(q)
        SR.check_span(net, gate, state=state, ws=ws, rows=audio[lo:hi], row0=lo, frame0=f0, n=n, pred_all=np.concatenate(preds),
                      params=q, noise=nz, uniform=un, pre=pre, sigma_scale=sigma)
    return gate, np.concatenate(params)


@pytest.mark.parametrize("name,over,nframe", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_stage_truths_compose_to_the_float64_incremental_emulator(name, over, nframe):
    """Each stage fed the previous stage's float64 value, h teacher-forced with the incremental emulator's own float64
    samples: the GMM parameters of every frame within 1e-9 relative."""
    opt = A.default_opt(**over)
    sd = A.make_state_dict(opt, "B", 3)
    net = SR.Net(opt, sd)
    audio, pre, noise, _ = _clip(opt, nframe)
    pred, params = INC.generate_incremental(sd, audio, pre, noise, opt, 0.3, return_params=True)
    ds1, _ = SR.ds1_stage(net, audio.astype(np.float64), "semantic")
    ds2, _ = SR.ds2_stage(net, ds1)
    cond = SR.cond_stage(net, ds2, "semantic")[0].reshape(len(audio), net.L, 2 * SR.R)
    rf, T = net.rf, net.rf - 1 + nframe
    X = np.zeros((net.L, T, SR.R))
    out = np.zeros_like(params)
    for t in range(T):
        h = pre.astype(np.float64) if t <= rf - 1 else pred[t - rf]
        x = SR.start_stage(net, h[None], SR.SLOPE)[0][0]
        ar = net.arow(np.array([t]), 0, len(audio))[0]
        skips = []
        for l, d in enumerate(net.dil):
            X[l, t] = x
            xd = X[l, t - d] if t - d >= 0 else np.zeros(SR.R)
            b = SR.block_stage(net, l, x[None], xd[None], cond[ar, l][None], SR.SLOPE)
            skips.append(b["skip"])
            x = b["out"][0]
        if t >= rf - 1:
            out[t - rf + 1] = SR.frame_stage(net, skips, [np.zeros_like(s) for s in skips], SR.SLOPE)[0][0]
    rel = np.abs(out - params).max() / np.abs(params).max()
    print(f"{name}: stage truths vs float64 incremental emulator, max rel {rel:.3g}")
    assert rel <= 1e-9


def test_fp32_emulator_matches_the_oracle():
    opt = A.default_opt()
    sd = A.make_state_dict(opt, "B", 3)
    net = SR.Net(opt, sd)
    audio, pre, noise, _ = _clip(opt, 40)
    gate, params = run_emulator(net, audio, pre, noise, None, 0.3)
    _, rp = A.generate_sequences(sd, audio, pre, noise, opt, 0.3, return_params=True)
    e = np.abs(params - rp).max()
    print(f"fp32 emulator vs oracle: max|params - oracle| = {e:.3g}")
    assert e <= 1e-4


@pytest.mark.parametrize("name,over,nframe", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_clean_emulator_stays_within_every_bound(name, over, nframe):
    opt = A.default_opt(**over)
    net = SR.Net(opt, A.make_state_dict(opt, "B", 3))
    audio, pre, noise, uniform = _clip(opt, nframe + 40)
    gate, _ = run_emulator(net, audio, pre, noise if net.gmm else None, uniform, 0.3, label=name)
    print("\n" + gate.report())
    assert not gate.failures, "\n".join(gate.failures[:10])
    assert {s for s, _ in gate.worst} == {"ds1", "ds2", "cond", "start", "block", "frame", "sample", "h"}


# defect -> (option overrides, what it plants)
DEFECT_CASES = {
    "tap": ({}, "block 3's delayed tap reads slot t - d + 1"),
    "arow": ({}, "the conditioning row is not clamped, so warm-up rows below 0 wrap to the clip's end"),
    "skip_bias": ({}, "the skip bias of a median-|bias| channel of one block is dropped"),
    "bn_shift": ({}, "the BatchNorm shift is folded without the linear layer's bias b0"),
    "gate_sign": ({}, "the gate uses 1 / (1 + exp(g))"),
    "rank_rows": ({}, "cluster rank 2's filter / gate channels use rank 3's weight rows"),
    "sigma_other": (dict(A2H_GMM_ncenter=2), "sigma is taken from the other mixture component"),
    "res_bias": ({}, "the residual bias of the smallest-|bias| channel of one block is dropped"),
    "h_fma": ({}, "the state's trailing sample is rounded once by a fused multiply-add, pred twice"),
}
SMALL = 1e-4       # the oracle tests' tolerance on the GMM parameters


def test_every_planted_defect_is_caught():
    """Each defect drives some stage past its bound; at least two of them move the GMM parameters by less than the
    1e-4 the oracle tests allow, so only the stage checks see them."""
    lines, small, missed = [], 0, []
    for defect, (over, what) in DEFECT_CASES.items():
        opt = A.default_opt(**over)
        net = SR.Net(opt, A.make_state_dict(opt, "B", 3))
        audio, pre, noise, uniform = _clip(opt, 40)
        _, clean = run_emulator(net, audio, pre, noise, uniform, 0.3)
        gate, params = run_emulator(net, audio, pre, noise, uniform, 0.3, defect=defect, label=defect)
        (stage, _), worst = max(gate.worst.items(), key=lambda kv: kv[1]["ratio"])
        dp = float(np.abs(params - clean).max())
        small += dp < SMALL
        if not worst["ratio"] > 1:
            missed.append(defect)
        lines.append(f"  {defect:<12s} worst err/bound {worst['ratio']:10.3g} at {stage:<6s} {worst['where']:<28s} "
                     f"max|dparams| {dp:.3g}   ({what})")
    print("\n" + "\n".join(lines) + f"\n  {small} of {len(DEFECT_CASES)} move the params by less than {SMALL:g}")
    assert not missed, missed
    assert small >= 2


@pytest.mark.parametrize("name,over", [(c[0], c[1]) for c in CONFIGS] + [("16x1", dict(A2H_wavenet_residual_layers=16, A2H_wavenet_residual_blocks=1)),
                                                                      ("in1", dict(A2H_wavenet_input_channels=1, A2H_GMM_ndim=1)),
                                                                      ("apc1024", dict(APC_hidden_size=1024, A2H_wavenet_cond_channels=1024))])
def test_state_and_workspace_layouts_on_a_host_only_handle(name, over):
    from livespeechportraits_b200 import _lib, headpose
    opt = A.default_opt(**over)
    cfg = headpose.config_from_opt(opt)
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.lsph_create(C.byref(h), C.byref(cfg), -1) == 0, lib.lsph_last_error()
    try:
        L, H = cfg.layers * cfg.blocks, cfg.apc_hidden
        got = C.c_size_t()
        assert lib.lsph_state_bytes(h, C.byref(got)) == 0
        assert got.value == 4 * (L * 2 ** cfg.layers * 128 + 32)
        pad = lambda k: (k + 63) // 64 * 64      # noqa: E731
        for n in (0, 1, 7, 65, 687):
            assert lib.lsph_stream_workspace_bytes(h, n, C.byref(got)) == 0
            assert got.value == 4 * (2 * pad(n * H) + pad(n * L * 2 * 128)), n
    finally:
        lib.lsph_destroy(h)
