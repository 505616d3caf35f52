"""Time live streaming through demo.py stages 1-4 (livespeechportraits_b200/stream.py) on the GPU.

    python tests/gpu_scripts/stream_bench.py [--repeats 3] [--profile-pushes 200]

00083.wav (tests/golden/mel/mel_00083_wav.npz, 183,296 samples) goes through ``AudioStream`` in one-video-frame pushes of
267 samples (16.7 ms of audio: the real-time budget of a push), with synthetic weights (rnn_oracle / a2h_oracle recipes
B) and a 10,000-row ``lle_oracle.make_database`` feature base.  Prints ONE JSON line with:
  * the wall time per push, host clock around ``push`` plus ``torch.cuda.synchronize()``: median, p99 and max over all
    pushes of ``--repeats`` streams (the first stream is a warm-up and not counted);
  * the total streamed time of the clip against the whole-clip chain (logmel -> APC -> projection -> mouth and head-pose
    generate), host clock with a synchronise at the end, medians of ``--repeats``;
  * from a separate run under torch.profiler: the kernel time per push, summed over every kernel, and the five kernels
    with the most time per push;
  * whether the streamed tracks equal the whole-clip tracks (torch.equal).
Card name and power limit come from a read-only nvidia-smi query in the same run.  Writes nothing.
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

from lle_bench import card  # noqa: E402
from livespeechportraits_b200.audio import MelFrontEnd  # noqa: E402
from livespeechportraits_b200.headpose import HeadposeGenerator, draw_reference_noise  # noqa: E402
from livespeechportraits_b200.manifold import ManifoldProjector  # noqa: E402
from livespeechportraits_b200.recurrent import ApcEncoder, MouthGenerator  # noqa: E402
from livespeechportraits_b200.stream import AudioStream  # noqa: E402
from oracle import a2h_oracle as A  # noqa: E402
from oracle import lle_oracle as M  # noqa: E402
from oracle import rnn_oracle as R  # noqa: E402

PUSH = 267


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--profile-pushes", type=int, default=200)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    name, limit = card()
    g = np.load(os.path.join(ROOT, "tests", "golden", "mel", "mel_00083_wav.npz"))
    audio = g["audio"]
    mopt, hopt = R.default_mouth_opt(), A.default_opt()
    stages = (MelFrontEnd(g["basis"], device=dev), ApcEncoder(R.make_apc_state_dict("B", 0), device=dev),
              MouthGenerator(mopt, R.make_mouth_state_dict(mopt, "B", 0), device=dev),
              HeadposeGenerator(hopt, A.make_state_dict(hopt, "B", 1), device=dev))
    proj = ManifoldProjector(M.make_database(10_000, 512, seed=1), device=dev)
    mel, apc, mouth, head = stages

    def whole():
        blend = proj.project_features(apc.forward(mel.logmel(audio)), 10, 1.0)
        torch.manual_seed(0)
        noise, _ = draw_reference_noise(blend.shape[0] // 2 - 15, 12, 1)
        return mouth.generate(blend), head.generate(blend.view(-1, 1024), np.zeros(12, np.float32), noise, 0.3)

    def streamed(times=None, limit_pushes=None):
        torch.manual_seed(0)
        s = AudioStream(mel, apc, mouth, head, projector=proj, k=10, percent=1.0, sigma_scale=0.3)
        ms, hs = [], []
        for j, at in enumerate(range(0, audio.shape[0], PUSH)):
            if limit_pushes is not None and j >= limit_pushes:
                return None
            t0 = time.perf_counter()
            r = s.push(audio[at:at + PUSH])
            torch.cuda.synchronize()
            if times is not None:
                times.append(time.perf_counter() - t0)
            ms.append(r.mouth)
            hs.append(r.headpose)
        r = s.finish()
        return torch.cat(ms + [r.mouth]), torch.cat(hs + [r.headpose])

    wm, wh = whole()
    sm, sh = streamed()
    torch.cuda.synchronize()
    equal = bool(torch.equal(wm, sm) and torch.equal(wh, sh))

    push_s, total_stream, total_whole = [], [], []
    for _ in range(a.repeats):
        t0 = time.perf_counter()
        whole()
        torch.cuda.synchronize()
        total_whole.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        streamed(push_s)
        torch.cuda.synchronize()
        total_stream.append(time.perf_counter() - t0)
    p = np.array(push_s) * 1e3

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        streamed(limit_pushes=a.profile_pushes)
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        t = getattr(ev, "device_time", None)
        t = (t if t is not None else getattr(ev, "cuda_time", 0.0)) / 1000.0
        if t > 0:
            per[ev.name] = per.get(ev.name, 0.0) + t
    n_prof = a.profile_pushes
    top = sorted(per.items(), key=lambda kv: -kv[1])[:5]

    print(json.dumps({
        "card": name, "power_limit": limit, "push_samples": PUSH, "pushes_per_stream": len(range(0, audio.shape[0], PUSH)),
        "budget_ms": 1000.0 * PUSH / 16000,
        "push_ms": {"median": float(np.median(p)), "p99": float(np.percentile(p, 99)), "max": float(p.max()), "n": int(p.size)},
        "clip_ms": {"streamed": 1e3 * float(np.median(total_stream)), "whole": 1e3 * float(np.median(total_whole))},
        "kernel_ms_per_push": sum(per.values()) / n_prof,
        "top_kernels_ms_per_push": {k[:80]: v / n_prof for k, v in top},
        "streamed_equals_whole": equal,
    }))


if __name__ == "__main__":
    main()
