"""The head-pose loop kernel (csrc/lsph.cu) checked stage by stage against float64 truths (tests/a2h_stage_reference.py),
at every emitted step, in the configurations lsph_create accepts, at cluster 1 and 8.

The clip runs through ``lsph_generate_stream`` in spans of at most ring / 2 frames with a test-owned state and
workspace; after each span both are copied back and every stage of every step among the span's last ring / 2 steps
is checked on the exact fp32 values it consumed: the hoisted GEMMs on the span's rows, the start convs, every
residual block, every frame's network output and its Sample_GMM draw.  The spans together cover every emitted step, and
their concatenation must equal one whole-clip ``generate`` bit for bit."""
from __future__ import annotations

import os
import sys
import time

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import a2h_stage_reference as SR  # noqa: E402
from oracle import a2h_oracle as A  # noqa: E402

pytestmark = pytest.mark.gpu

# (name, option overrides, recipe, frames, clusters, seeded subset of steps per span or None)
CASES = [
    ("default-A-1", {}, "A", 1, (1, 8), None),
    ("default-B-1", {}, "B", 1, (1, 8), None),
    ("default-A-65", {}, "A", 65, (1, 8), None),
    ("default-B-65", {}, "B", 65, (1, 8), None),
    ("default-A-672", {}, "A", 672, (1, 8), None),
    ("default-B-672", {}, "B", 672, (1, 8), None),
    ("8x2", dict(A2H_wavenet_residual_layers=8), "B", 300, (1, 8), None),
    ("4x4", dict(A2H_wavenet_residual_layers=4, A2H_wavenet_residual_blocks=4), "B", 100, (1, 8), None),
    ("1x16", dict(A2H_wavenet_residual_layers=1, A2H_wavenet_residual_blocks=16), "B", 24, (1, 8), None),
    ("16x1", dict(A2H_wavenet_residual_layers=16, A2H_wavenet_residual_blocks=1), "B", 20, (1, 8), 160),
    ("ncenter5", dict(A2H_GMM_ncenter=5), "B", 100, (1, 8), None),
    ("in1", dict(A2H_wavenet_input_channels=1, A2H_GMM_ndim=1), "B", 100, (1, 8), None),
    ("in32", dict(A2H_wavenet_input_channels=32, A2H_GMM_ndim=32), "B", 100, (1, 8), None),
    ("L2", dict(loss="L2"), "B", 100, (1, 8), None),
    ("no_bias", dict(A2H_wavenet_use_bias=False), "B", 100, (1, 8), None),
    ("ff0", dict(frame_future=0), "B", 100, (1, 8), None),
    ("apc64", dict(APC_hidden_size=64, A2H_wavenet_cond_channels=64), "B", 100, (1, 8), None),
    ("apc1024", dict(APC_hidden_size=1024, A2H_wavenet_cond_channels=1024), "B", 100, (1, 8), None),
]
PARAMS = [(c, cl) for c in CASES for cl in c[4]] + [(("long-B-36000", {}, "B", 36000, (8,), None), 8)]


def _drive(case, cluster):
    from livespeechportraits_b200.headpose import HeadposeGenerator
    name, over, recipe, nframe, _, subset = case
    opt = A.default_opt(**over)
    sd = A.make_state_dict(opt, recipe, 3)
    net = SR.Net(opt, sd)
    gen = HeadposeGenerator(opt, sd, device=torch.device("cuda", 0))
    dev = gen.device
    audio = A.make_audio_feats(nframe + net.ff, opt, 4)
    pre = np.linspace(-0.3, 0.2, net.I).astype(np.float32)
    rng = np.random.Generator(np.random.PCG64(11))
    noise = rng.standard_normal((nframe, net.ndim)).astype(np.float32) if net.gmm else None
    uniform = rng.uniform(0.0, 1.0, nframe).astype(np.float32) if net.nc > 1 else None
    ad = torch.from_numpy(audio).to(dev)
    pre_d = torch.from_numpy(pre).to(dev)
    nz_d = torch.from_numpy(noise).to(dev) if noise is not None else torch.zeros((nframe, net.ndim), device=dev)
    un_d = torch.from_numpy(uniform).to(dev) if uniform is not None else None
    whole_pred, whole_params = gen.generate(ad, pre_d, nz_d, 0.3, uniform=un_d, return_params=True, cluster=cluster)
    whole_pred, whole_params = whole_pred.cpu().numpy(), whole_params.cpu().numpy()

    state = gen._new_state()
    ws = None
    plan = SR.span_plan(net, nframe)
    check = set(range(len(plan)))
    if nframe > 5000:       # the first, the last and a seeded eighth of the spans
        pick = np.random.Generator(np.random.PCG64(5)).choice(len(plan), len(plan) // 8, replace=False)
        check = {0, len(plan) - 1} | set(int(i) for i in pick)
    gate = SR.Gate(f"{name} cl{cluster}")
    preds, params = [], []
    for si, (f0, n) in enumerate(plan):
        lo, hi = SR.span_rows(net, f0, n)
        un = un_d[f0:f0 + n].contiguous() if un_d is not None else None
        p, q, ws = gen._run(ad[lo:hi].contiguous(), lo, f0, n, pre_d, nz_d[f0:f0 + n].contiguous(), un, 0.3, state, ws, True, cluster)
        preds.append(p.cpu().numpy())
        params.append(q.cpu().numpy())
        if si not in check:
            continue
        st = state.cpu().numpy()
        _, need = net.ws_offsets(hi - lo)
        wsh = ws.view(torch.float32)[:need].cpu().numpy()                   # a byte buffer (_lib.reserve)
        steps = None
        if subset:
            t_end = f0 + n + net.rf - 2
            lo_t = max(0 if f0 == 0 else f0 + net.rf - 1, t_end - net.ring // 2 + 1)
            r = np.random.Generator(np.random.PCG64(7 + si))
            emit = np.arange(max(lo_t, net.rf - 1), t_end + 1)
            steps = set(emit.tolist()) | set(r.integers(lo_t, t_end + 1, subset).tolist())
        SR.check_span(net, gate, state=st, ws=wsh, rows=audio[lo:hi], row0=lo, frame0=f0, n=n, pred_all=np.concatenate(preds),
                      params=params[-1], noise=noise[f0:f0 + n] if noise is not None else None,
                      uniform=uniform[f0:f0 + n] if uniform is not None else None, pre=pre, sigma_scale=0.3, steps=steps)
    pred_s, params_s = np.concatenate(preds), np.concatenate(params)
    return net, gate, pred_s, params_s, whole_pred, whole_params


@pytest.mark.parametrize("case,cluster", PARAMS, ids=[f"{c[0]}-cl{cl}" for c, cl in PARAMS])
def test_every_stage_of_every_step_against_float64(case, cluster):
    t0 = time.time()
    net, gate, pred_s, params_s, whole_pred, whole_params = _drive(case, cluster)
    assert np.array_equal(pred_s, whole_pred) and np.array_equal(params_s, whole_params), "spans differ from the whole clip"
    fr = gate.worst[("frame", "kernel")]
    print(f"\n{case[0]} cluster {cluster}: {time.time() - t0:.1f} s; params bound {fr['min_bound']:.3g} .. {fr['bound']:.3g} "
          f"(old gate 1e-4)\n" + gate.report())
    assert not gate.failures, "\n".join(gate.failures[:20])
