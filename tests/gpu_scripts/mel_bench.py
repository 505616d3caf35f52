"""Time the log-mel front end (row N6) on the GPU against the reference's per-window loop.

    python tests/gpu_scripts/mel_bench.py [--iters 50] [--cpu-reps 3]

Prints ONE JSON line.  For the shipped clip (00083.wav, 1374 windows, from the golden fixture) and a 10-minute synthetic
clip (72k windows): the kernel time from torch.profiler (lspa_logmel_kernel, mean over --iters calls after warm-up), the
CUDA-event time of MelFrontEnd.logmel on device-resident audio, and the wall time of the installed drop-in
compute_mel_one_sequence (handle creation, basis and audio upload and result download included).  For the shipped clip
also the oracle restatement of the reference loop (same torch calls, one window per call) on the host cores and with the
clips on cuda:0 as ``device='cuda'`` runs it.  Card name and power limit come from a read-only nvidia-smi query.  Writes
nothing.
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
from livespeechportraits_b200 import audio as A  # noqa: E402
from oracle import mel_oracle as O  # noqa: E402


def kernel_ms(fn, iters):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    total = 0.0
    for ev in prof.events():
        if "lspa_logmel_kernel" in ev.name:
            t = getattr(ev, "device_time", None)
            total += (t if t is not None else getattr(ev, "cuda_time", 0.0)) / 1000.0
    return total / iters


def oracle_loop_ms(audio, basis, device, reps):
    """The reference loop restated (oracle/mel_oracle.py audio2mel per window), clips and basis on ``device``."""
    b = torch.from_numpy(basis).to(device)
    starts = O.window_starts(O.n_windows(len(audio)), 16000 * 0.5 / 60)
    best = float("inf")
    for _ in range(reps):
        t0 = time.perf_counter()
        out = np.zeros([len(starts), 80])
        for i, st in enumerate(starts):
            c = torch.from_numpy(O.clip(audio, int(st), 266))[None, None, :].to(device)
            out[i] = O.audio2mel(c, b).cpu().numpy()[0].T
        best = min(best, (time.perf_counter() - t0) * 1e3)
    return best


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--cpu-reps", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    name, limit = card()
    basis = O.make_basis(80)
    front = A.MelFrontEnd(basis, device=dev)
    res = {"card": name, "power_limit": limit, "cpu_threads": torch.get_num_threads(), "clips": {}}
    for label, clip in (("00083.wav", O.read_wav_fixture()), ("10 min synthetic", O.make_audio(600 * 16000, 1))):
        x = torch.from_numpy(clip).to(dev)
        for _ in range(3):
            front.logmel(x)
        torch.cuda.synchronize()
        walls = []
        for _ in range(5):
            t0 = time.perf_counter()
            A.compute_mel_one_sequence(clip, device="cuda")
            walls.append((time.perf_counter() - t0) * 1e3)
        r = {"windows": O.n_windows(len(clip)),
             "kernel_ms": round(kernel_ms(lambda: front.logmel(x), a.iters), 4),
             "logmel_call_ms": round(event_ms(lambda: front.logmel(x), a.iters), 4),
             "dropin_wall_ms_incl_upload_download": round(min(walls), 2)}
        if label == "00083.wav":
            r["oracle_loop_cpu_ms"] = round(oracle_loop_ms(clip, basis, torch.device("cpu"), a.cpu_reps), 1)
            r["oracle_loop_device_cuda_ms"] = round(oracle_loop_ms(clip, basis, dev, a.cpu_reps), 1)
        res["clips"][label] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
