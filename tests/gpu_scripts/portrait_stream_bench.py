"""Time live portraits (livespeechportraits_b200/stream.py ``PortraitStream``: audio in, frames out) on the GPU.

    python tests/gpu_scripts/portrait_stream_bench.py [--repeats 2] [--profile-pushes 200]

00083.wav (tests/golden/mel/mel_00083_wav.npz) goes through a ``PortraitStream`` in one-video-frame pushes of 267
samples (16.7 ms of audio: the real-time budget of a push), with synthetic weights (rnn_oracle / a2h_oracle recipes B,
f2f_oracle ``large`` recipe B), a 10,000-row ``lle_oracle.make_database`` feature base, May's stage-5 settings and the
``large`` generator at 512 x 512 in parity mode.  Prints ONE JSON line with:
  * the wall time per push, host clock around ``push`` plus ``torch.cuda.synchronize()``: median, p99 and max over all
    pushes of ``--repeats`` streams (a first stream is a warm-up and not counted), and the frames out per push;
  * from a separate run under torch.profiler: the kernel time per push split into stages 1-4, stage 5 (lspl_*), the
    rasteriser and the generator, plus torch's own copy / concatenation kernels;
  * the look-ahead in video frames (``portrait_counts``);
  * the cost of the live lip fix's sequential sum on a whole 36,000-frame clip pushed at once, against ``run``
    (CUDA events, median of 5).
Card name and power limit come from a read-only nvidia-smi query in the same run.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from lle_bench import card  # noqa: E402
from livespeechportraits_b200.audio import MelFrontEnd  # noqa: E402
from livespeechportraits_b200.generator import Feature2Face_G  # noqa: E402
from livespeechportraits_b200.headpose import HeadposeGenerator  # noqa: E402
from livespeechportraits_b200.landmarks import Identity, LandmarkPostprocessor, StageParams  # noqa: E402
from livespeechportraits_b200.manifold import ManifoldProjector  # noqa: E402
from livespeechportraits_b200.recurrent import ApcEncoder, MouthGenerator  # noqa: E402
from livespeechportraits_b200.stream import AudioStream, PortraitStream, portrait_counts  # noqa: E402
from oracle import a2h_oracle as A  # noqa: E402
from oracle import f2f_oracle as F  # noqa: E402
from oracle import landmark_oracle as O  # noqa: E402
from oracle import lle_oracle as M  # noqa: E402
from oracle import rnn_oracle as R  # noqa: E402

PUSH = 267
STAGE14 = ("lspa", "logmel", "rnn_layer", "lspr", "headpose", "lsph", "lspm", "knn", "lle", "gemm_nt")


def kind(name: str) -> str:
    if "lspl_" in name:
        return "stage5"
    if "raster" in name:
        return "raster"
    if any(k in name for k in STAGE14):
        return "stages1_4"
    if "at::" in name or "Memcpy" in name or "Memset" in name or "elementwise" in name or "CatArray" in name:
        return "torch_copies"
    return "generator"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--profile-pushes", type=int, default=200)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    name, limit = card()
    g = np.load(os.path.join(ROOT, "tests", "golden", "mel", "mel_00083_wav.npz"))
    audio = g["audio"]
    mopt, hopt = R.default_mouth_opt(), A.default_opt()
    mel, apc = MelFrontEnd(g["basis"], device=dev), ApcEncoder(R.make_apc_state_dict("B", 0), device=dev)
    mouth = MouthGenerator(mopt, R.make_mouth_state_dict(mopt, "B", 0), device=dev)
    head = HeadposeGenerator(hopt, A.make_state_dict(hopt, "B", 1), device=dev)
    proj = ManifoldProjector(M.make_database(10_000, 512, seed=1), device=dev)
    net = Feature2Face_G(types.SimpleNamespace(isTrain=False, size="large", n_downsample_G=8, ngf=64, fp16=0),
                         precision="parity")
    net.load_state_dict(F.make_state_dict("large", "B"))
    net = net.to(dev).eval()
    _, cand = F.make_inputs(1, 512, 512, seed=6)
    cand = cand[:1].to(dev)
    ident = O.make_identity(0, 37)
    post = LandmarkPostprocessor(Identity(**ident), device=dev)
    p = O.MAY
    params = StageParams(p["Feat_smooth_sigma"], p["AMP_method"], p["Feat_AMPs"], p["rot_AMP"], p["trans_AMP"],
                         p["Head_smooth_sigma"], p["shoulder_AMP"])

    def session(times=None, counts=None, limit_pushes=None):
        torch.manual_seed(0)
        s = PortraitStream(AudioStream(mel, apc, mouth, head, projector=proj, k=10, percent=1.0, sigma_scale=0.3), post,
                           params, net, cand, size=(512, 512))
        for j, at in enumerate(range(0, audio.shape[0], PUSH)):
            if limit_pushes is not None and j >= limit_pushes:
                return
            t0 = time.perf_counter()
            r = s.push(audio[at:at + PUSH])
            torch.cuda.synchronize()
            if times is not None:
                times.append(time.perf_counter() - t0)
                counts.append(r.frames.shape[0])
        s.finish()
        torch.cuda.synchronize()

    session()
    push_s, outs = [], []
    for _ in range(a.repeats):
        session(push_s, outs)
    ms = np.array(push_s) * 1e3
    steady = ms[np.array(outs) > 0]

    from torch.profiler import ProfilerActivity, profile
    session(limit_pushes=a.profile_pushes)                    # warm for the profiled pushes
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        session(limit_pushes=a.profile_pushes)
        torch.cuda.synchronize()
    split = {}
    for ev in prof.events():
        t = getattr(ev, "device_time", None)
        t = (t if t is not None else getattr(ev, "cuda_time", 0.0)) / 1000.0
        if t > 0:
            k = kind(ev.name)
            split[k] = split.get(k, 0.0) + t

    # the live lip fix's sequential sum over a whole clip pushed at once, against run
    feat, hd = O.make_tracks(36000, 36010, 41)
    f, h = torch.from_numpy(feat).to(dev), torch.from_numpy(hd).to(dev)

    def timed(fn):
        out = []
        for _ in range(6):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            out.append(e0.elapsed_time(e1))
        return float(np.median(out[1:]))

    def whole_push():
        s = post.stream(params)
        s.push(f, h)
        s.finish()
    run_ms, stream_ms = timed(lambda: post.run(f, h, params)), timed(whole_push)

    first = next(n for n in range(0, 100000, 1) if portrait_counts(n, False, params) > 0)
    print(json.dumps({
        "card": name, "power_limit": limit, "push_samples": PUSH, "budget_ms": 1000.0 * PUSH / 16000,
        "generator": "large 512x512 parity",
        "push_ms_all": {"median": float(np.median(ms)), "p99": float(np.percentile(ms, 99)), "max": float(ms.max()),
                        "n": int(ms.size)},
        "push_ms_with_frames": {"median": float(np.median(steady)), "p99": float(np.percentile(steady, 99)),
                                "n": int(steady.size)},
        "frames_per_push": {str(k): int(v) for k, v in zip(*np.unique(outs, return_counts=True))},
        "kernel_ms_per_push": {k: v / a.profile_pushes for k, v in sorted(split.items())},
        "lookahead": {"first_frame_after_samples": first, "frames": int(round(first / PUSH))},
        "clip36000_ms": {"run": run_ms, "stream_one_push": stream_ms},
    }))


if __name__ == "__main__":
    main()
