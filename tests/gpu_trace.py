"""Dump the in-kernel clock64 trace of conv layers (debug tool; see conv_wgmma.cuh kTraceSlots).
    LSPG_TRACE_LAYERS=<i,j,...> [LSPG_TRACE_SKIP=<first local tile>] python tests/gpu_trace.py <variant> <mode> <B>
One process, one generator instance per traced layer (the trace target is fixed when the launch plan is built)."""
import os
import statistics
import sys
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from oracle import f2f_oracle as O
from livespeechportraits_b200 import _lib
from livespeechportraits_b200.generator import Feature2Face_G

variant, mode, B = sys.argv[1], sys.argv[2], int(sys.argv[3])
os.environ["LSPG_NO_GRAPH"] = "1"
layers = [int(v) for v in os.environ.get("LSPG_TRACE_LAYERS", os.environ.get("LSPG_TRACE_LAYER", "1")).split(",")]
sd = O.make_state_dict(variant, "A")
fm, cand = O.make_inputs(B, 512, 512)
x = torch.cat([fm, cand], 1).cuda()
SLOTS, TILES = 4 + 8 * 12 + 4, 12
show_ctas = [int(v) for v in os.environ.get("LSPG_TRACE_CTAS", "0,1,73,147").split(",")]

for layer in layers:
    os.environ["LSPG_TRACE_LAYER"] = str(layer)
    net = Feature2Face_G(types.SimpleNamespace(isTrain=False, size=variant, n_downsample_G=8, ngf=64, fp16=0), precision=mode)
    net.load_state_dict(sd)
    net = net.cuda().eval()
    for _ in range(3):
        net(x)
    torch.cuda.synchronize()
    buf = np.zeros(256 * SLOTS, np.uint64)
    _lib.check(net._lib.lspg_debug_read_trace(net._handle, buf.ctypes.data, buf.size))
    t = buf.reshape(256, SLOTS).astype(np.int64)
    row = net.layer_table(512, 512)[layer]
    print(f"layer {layer}: {row}")
    starts = [int(t[c][0]) for c in range(256) if t[c][0]]
    if not starts:
        print("  (no trace: this layer's kernel has no stamps)")
        continue
    print(f"  CTAs {len(starts)}")
    for cta in show_ctas:
        e = t[cta]
        if e[0] and e[3] > e[2]:
            cyc, ns = int(e[4 + 8 * TILES] - e[0]), int(e[3] - e[2])
            print(f"  CTA {cta}: lifetime {cyc} cyc = {ns} ns -> SM clock {cyc / ns:.3f} GHz")
    for cta in show_ctas:
        e = t[cta]
        if e[0] == 0:
            continue
        t0 = e[0]
        print(f"CTA {cta}: prologue {e[1] - t0} cyc")
        for i in range(TILES):
            s = e[4 + 8 * i: 12 + 8 * i]
            if not s.any():
                break
            rel = [int(v - t0) if v else -1 for v in s]
            print(f"   tile {i}: start {rel[0]:7d} first_stage {rel[1]:7d} mma_done {rel[2]:7d} epi_done {rel[3]:7d} "
                  f"| prod_first {rel[6]:7d} prod_last {rel[7]:7d}")
    spans = {"wait_first_stage": [], "mma": [], "epi": [], "total": []}
    for cta in range(256):
        e = t[cta]
        if e[0] == 0:
            continue
        last = 0
        for i in range(TILES):
            s = e[4 + 8 * i: 12 + 8 * i]
            if s[3] == 0:
                break
            spans["wait_first_stage"].append(int(s[1] - s[0]))
            spans["mma"].append(int(s[2] - s[1]))
            spans["epi"].append(int(s[3] - s[2]))
            last = max(last, int(s[3] - e[0]))
        spans["total"].append(last)
    for k, v in spans.items():
        if v:
            print(f"{k}: n={len(v)} mean={statistics.mean(v):.0f} median={statistics.median(v):.0f} max={max(v)}")
    del net
    torch.cuda.empty_cache()
