"""Time the landmark post-processing (row N7, demo.py stage 5) on the GPU against the reference's numpy stage.

    python tests/gpu_scripts/landmark_bench.py [--iters 50] [--cpu-reps 3]

Prints ONE JSON line.  For a 672-frame clip (May's parameters) and a 36,000-frame (10-minute) clip: the kernel times from
torch.profiler (lspl_smooth_kernel and lspl_project_kernel, mean over --iters calls after warm-up), the CUDA-event time of
LandmarkPostprocessor.run on device-resident tracks, and the wall time of postprocess_clip (handle creation, identity,
track upload and result download included).  For the 672-frame clip also the oracle restatement of demo.py:217-255
(oracle/landmark_oracle.py stage5: scipy and the two per-frame loops) on the host cores.  Card name and power limit come
from a read-only nvidia-smi query.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from lle_bench import card, event_ms  # noqa: E402
from livespeechportraits_b200 import landmarks as L  # noqa: E402
from oracle import landmark_oracle as O  # noqa: E402


def kernel_ms(fn, iters):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    total = {"lspl_smooth_kernel": 0.0, "lspl_project_kernel": 0.0}
    for ev in prof.events():
        for k in total:
            if k in ev.name:
                t = getattr(ev, "device_time", None)
                total[k] += (t if t is not None else getattr(ev, "cuda_time", 0.0)) / 1000.0
    return {k: round(v / iters, 4) for k, v in total.items()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--cpu-reps", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    name, limit = card()
    ident = O.make_identity(0)
    prm = O.MAY
    params = L.StageParams(*(prm[k] for k in ("Feat_smooth_sigma", "AMP_method", "Feat_AMPs", "rot_AMP", "trans_AMP",
                                              "Head_smooth_sigma", "shoulder_AMP")))
    post = L.LandmarkPostprocessor(L.Identity(**ident), device=dev)
    res = {"card": name, "power_limit": limit, "cpu_threads": torch.get_num_threads(), "clips": {}}
    for n in (672, 36000):
        feat, head = O.make_tracks(n, n, 1)
        f, h = torch.from_numpy(feat).to(dev), torch.from_numpy(head).to(dev)
        for _ in range(3):
            post.run(f, h, params)
        torch.cuda.synchronize()
        walls = []
        for _ in range(5):
            t0 = time.perf_counter()
            L.postprocess_clip(feat, head, *(ident[k] for k in O.IDENTITY_KEYS), *(prm[k] for k in (
                "Feat_smooth_sigma", "AMP_method", "Feat_AMPs", "rot_AMP", "trans_AMP", "Head_smooth_sigma", "shoulder_AMP")))
            walls.append((time.perf_counter() - t0) * 1e3)
        r = {"frames": n, "kernel_ms": kernel_ms(lambda: post.run(f, h, params), a.iters),
             "run_call_ms": round(event_ms(lambda: post.run(f, h, params), a.iters), 4),
             "postprocess_clip_wall_ms": round(min(walls), 2)}
        if n == 672:
            best = float("inf")
            for _ in range(a.cpu_reps):
                t0 = time.perf_counter()
                O.stage5(feat, head, ident, prm)
                best = min(best, (time.perf_counter() - t0) * 1e3)
            r["oracle_stage5_host_ms"] = round(best, 1)
        res["clips"][str(n)] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
