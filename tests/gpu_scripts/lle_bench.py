"""Time the APC manifold projection (row N5) on the GPU against the reference's own host computation.

    python tests/gpu_scripts/lle_bench.py [--rows 1374] [--k 10] [--sizes 10000,30000,100000] [--iters 20]

Prints ONE JSON line.  Per database size N: the per-kernel GPU times from torch.profiler (lspm_norms_kernel,
lspm_knn_kernel, lspm_knn_merge_kernel, lspm_lle_kernel; means over --iters calls after warm-up), CUDA-event times of the
device-level knn() and project() calls, the wall time of the installed drop-ins (KNN_with_torch +
compute_LLE_projection_all_frame, database upload and result download included), and the CPU arm: the oracle restatement
of the reference (same torch / numpy calls, host cores).  The distance kernel's achieved rate is 2 n N dim / time, set
against the H100 SXM data-sheet fp32 (non-tensor) peak of 67 TFLOP/s.  Card name and power limit come from a read-only
nvidia-smi query.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from livespeechportraits_b200 import manifold  # noqa: E402
from oracle import lle_oracle as L  # noqa: E402

FP32_PEAK_DATASHEET = 67e12
KERNELS = ("lspm_norms_kernel", "lspm_knn_kernel", "lspm_knn_merge_kernel", "lspm_lle_kernel")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        name, limit = (s.strip() for s in out[0].split(","))
        return name, limit
    except Exception as exc:                        # the timing is still valid without the label
        return f"unknown ({exc})", "unknown"


def kernel_times(fn, iters):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    ms = {k: 0.0 for k in KERNELS}
    for ev in prof.events():
        t = getattr(ev, "device_time", None)
        if t is None:
            t = getattr(ev, "cuda_time", 0.0)
        for k in KERNELS:
            if k + "<" in ev.name or k + "(" in ev.name or ev.name.endswith(k):
                ms[k] += t / 1000.0
    return {k: v / iters for k, v in ms.items()}


def event_ms(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1374)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--dim", type=int, default=512)
    ap.add_argument("--sizes", default="10000,30000,100000")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--cpu-reps", type=int, default=1)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    name, limit = card()
    res = {"workload": f"{a.rows} rows x dim {a.dim}, K={a.k}", "card": name, "power_limit": limit,
           "fp32_peak_datasheet_tflops": FP32_PEAK_DATASHEET / 1e12, "sizes": {}}
    for N in (int(s) for s in a.sizes.split(",")):
        db = L.make_database(N, a.dim, 1)
        q = L.make_queries(a.rows, a.dim, 2, db)
        proj = manifold.ManifoldProjector(db, device=dev)
        qd = torch.from_numpy(q).to(dev)
        ind = proj.knn(qd, a.k)
        for _ in range(3):                                          # warm-up
            proj.project(qd, proj.knn(qd, a.k))
        torch.cuda.synchronize()
        kt = kernel_times(lambda: proj.project(qd, proj.knn(qd, a.k)), a.iters)
        knn_ms = event_ms(lambda: proj.knn(qd, a.k), a.iters)
        proj_ms = event_ms(lambda: proj.project(qd, ind), a.iters)
        walls = []
        for _ in range(3):
            t0 = time.perf_counter()
            i2 = manifold.KNN_with_torch(q, db, K=a.k)
            manifold.compute_LLE_projection_all_frame(q, db, i2, a.rows)
            walls.append((time.perf_counter() - t0) * 1e3)
        cpu_knn, cpu_lle = [], []
        for _ in range(a.cpu_reps):
            t0 = time.perf_counter()
            ci = L.knn_with_torch(q, db, a.k)
            t1 = time.perf_counter()
            L.compute_lle_projection_all(q, db, ci)
            t2 = time.perf_counter()
            cpu_knn.append((t1 - t0) * 1e3)
            cpu_lle.append((t2 - t1) * 1e3)
        flops = 2.0 * a.rows * N * a.dim
        knn_k = kt["lspm_knn_kernel"]
        res["sizes"][str(N)] = {
            "gpu_kernel_ms": {k: round(v, 4) for k, v in kt.items()},
            "gpu_knn_call_ms": round(knn_ms, 4), "gpu_project_call_ms": round(proj_ms, 4),
            "dropin_wall_ms_incl_upload_download": round(min(walls), 2),
            "cpu_reference_knn_ms": round(min(cpu_knn), 1), "cpu_reference_lle_ms": round(min(cpu_lle), 1),
            "knn_kernel_tflops": round(flops / (knn_k * 1e-3) / 1e12, 2) if knn_k > 0 else None,
            "knn_kernel_fraction_of_fp32_datasheet_peak": round(flops / (knn_k * 1e-3) / FP32_PEAK_DATASHEET, 3) if knn_k > 0 else None,
        }
        del proj
    res["cpu_threads"] = torch.get_num_threads()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
