"""GPU bring-up tool.

    python tests/gpu_bringup.py <stage> [variant] [recipe] [mode] [H] [B]

stage "final": compare the final image with the oracle.   stage "time": quick timing.
Per-layer checks of every conv launch are tests/test_gpu_layers.py.
"""
from __future__ import annotations

import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch  # noqa: E402

from oracle import f2f_oracle as O  # noqa: E402
from livespeechportraits_b200.generator import Feature2Face_G  # noqa: E402


def make_net(variant, recipe, mode):
    opt = types.SimpleNamespace(isTrain=False, size=variant, n_downsample_G=8, ngf=64, fp16=0)
    net = Feature2Face_G(opt, precision=mode)
    sd = O.make_state_dict(variant, recipe)
    net.load_state_dict(sd, strict=True)
    return net.cuda().eval(), sd


def stage_final(variant, recipe, mode, H, B):
    net, sd = make_net(variant, recipe, mode)
    fm, cand = O.make_inputs(B, H, H)
    x = torch.cat([fm, cand], 1)
    ref = O.generator_forward(sd, x, variant)
    out = net(x.cuda()).cpu()
    print(f"{variant} {recipe} {mode} {H} B{B}: max|out-oracle| = {(out - ref).abs().max().item():.4g} "
          f"(ref std {ref.std().item():.3f})", flush=True)
    out2 = net.render(fm.cuda(), cand[:1].cuda()).cpu()
    print(f"   split-input/broadcast-cand path differs from cat path by {(out2 - out).abs().max().item():.3g}")
    return 0


def stage_time(variant, recipe, mode, H, B):
    net, sd = make_net(variant, recipe, mode)
    fm, cand = O.make_inputs(B, H, H)
    x = torch.cat([fm, cand], 1).cuda()
    for _ in range(3):
        net(x)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 10
    e0.record()
    for _ in range(n):
        net(x)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    fl = net.flops_per_frame(H, H) * B
    print(f"{variant} {mode} {H} B{B}: {ms:.3f} ms/forward, {B / ms * 1e3:.1f} fps, {fl / ms / 1e9:.1f} TFLOP/s algorithmic",
          flush=True)
    if os.environ.get("LSPG_PER_LAYER"):
        net.profile_enable(True)
        for _ in range(n):
            net(x)
        torch.cuda.synchronize()
        t, cnt = net.profile_read()
        net.profile_enable(False)
        rows = net.layer_table(H, H)
        print(f"  pack_input {t[0] * 1e3:8.1f} us")
        for i, (r, v) in enumerate(zip(rows, t[1:])):
            print(f"  L{i:02d} k{r['kind']} {r['cin']:4d}->{r['cout']:3d} @{r['out_h']:3d} {v * 1e3:8.1f} us  "
                  f"{r['flops'] * B / (v * 1e-3) / 1e12:7.1f} TF/s alg")
    return 0


if __name__ == "__main__":
    stage = sys.argv[1]
    variant = sys.argv[2] if len(sys.argv) > 2 else "normal"
    recipe = sys.argv[3] if len(sys.argv) > 3 else "B"
    mode = sys.argv[4] if len(sys.argv) > 4 else "fast"
    H = int(sys.argv[5]) if len(sys.argv) > 5 else 256
    B = int(sys.argv[6]) if len(sys.argv) > 6 else 1
    print(f"=== {stage} {variant} {recipe} {mode} H={H} B={B} on {torch.cuda.get_device_name(0)}", flush=True)
    sys.exit({"final": stage_final, "time": stage_time}[stage](variant, recipe, mode, H, B))
