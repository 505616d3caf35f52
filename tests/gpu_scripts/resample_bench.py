"""Time librosa.load's resampling on the GPU (livespeechportraits_b200/audio.py ``Resampler``; csrc/lspa.cu
``lspa_resample_kernel``).

    python tests/gpu_scripts/resample_bench.py [--host]

Prints ONE JSON line with:
  * kernel time (CUDA events around ``lspa_resample_at``, median of 5 after a warm-up) for the 00083.wav duration
    (11.456 s) and for 10 minutes, at 44.1 and 48 kHz, ``kaiser_best``, fp32 mono and PCM16 stereo input;
  * the taps each clip needs, counted from shapes (both wings of every output, as resample_f runs them), and taps/s;
  * the wall time of a one-video-frame ``PortraitStream`` push (host clock around ``push`` plus a device synchronise),
    median and p99, for a stream fed 48 kHz PCM16 stereo (800 frames per push) and one fed 16 kHz fp32 (267 samples),
    their pushes alternated in one run; synthetic weights, a 10k-row feature base, May's settings, ``large`` at 512^2;
  * with ``--host``: the numpy restatement (oracle/resample_oracle.py) on the host cores for the 11.456 s clip at 48 kHz,
    labelled as such.  resampy itself (numba) is not installed and is not measured.
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
from livespeechportraits_b200.audio import MelFrontEnd, Resampler, register_at  # noqa: E402
from oracle import resample_oracle as RO  # noqa: E402

CLIP_S = 183296 / 16000


def taps(rs: Resampler, n_in: int) -> int:
    """Taps of the outputs of an n_in-frame clip: (nwin - offset) // index_step per wing, clamped at the clip's ends as resample_f
    clamps them (the kernel reads zeros there instead; the count is the reference's)."""
    nwin, step, num_table = rs.nwin, rs.index_step, rs.num_table
    scale = min(1.0, rs.sample_ratio)
    n_out = rs.n_out(n_in)
    total = 0
    for lo in range(0, n_out, 1 << 22):
        t = np.arange(lo, min(n_out, lo + (1 << 22)))
        reg = register_at(rs._reg, t)
        n = reg.astype(np.int64)
        frac = scale * (reg - n)
        left = (nwin - (frac * num_table).astype(np.int64)) // step
        right = (nwin - ((scale - frac) * num_table).astype(np.int64)) // step
        total += int(np.minimum(n + 1, left).sum() + np.maximum(0, np.minimum(n_in - n - 1, right)).sum())
    return total


def kernel_ms(rs: Resampler, frames: torch.Tensor, n_out: int) -> float:
    out = torch.empty(n_out, dtype=torch.float32, device=rs.device)
    times = []
    for _ in range(6):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rs._span(frames, 0, 0, n_out, out)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return float(np.median(times[1:]))


def live_pushes(dev, n_pushes: int):
    from livespeechportraits_b200.generator import Feature2Face_G
    from livespeechportraits_b200.headpose import HeadposeGenerator
    from livespeechportraits_b200.landmarks import Identity, LandmarkPostprocessor, StageParams
    from livespeechportraits_b200.manifold import ManifoldProjector
    from livespeechportraits_b200.recurrent import ApcEncoder, MouthGenerator
    from livespeechportraits_b200.stream import AudioStream, PortraitStream
    from oracle import a2h_oracle as A
    from oracle import f2f_oracle as F
    from oracle import landmark_oracle as O
    from oracle import lle_oracle as M
    from oracle import mel_oracle as W
    from oracle import rnn_oracle as R
    mopt, hopt = R.default_mouth_opt(), A.default_opt()
    mel, apc = MelFrontEnd(W.make_basis(80), device=dev), ApcEncoder(R.make_apc_state_dict("B", 0), device=dev)
    mouth = MouthGenerator(mopt, R.make_mouth_state_dict(mopt, "B", 0), device=dev)
    head = HeadposeGenerator(hopt, A.make_state_dict(hopt, "B", 1), device=dev)
    proj = ManifoldProjector(M.make_database(10_000, 512, seed=1), device=dev)
    net = Feature2Face_G(types.SimpleNamespace(isTrain=False, size="large", n_downsample_G=8, ngf=64, fp16=0),
                         precision="parity")
    net.load_state_dict(F.make_state_dict("large", "B"))
    net = net.to(dev).eval()
    cand = F.make_inputs(1, 512, 512, seed=6)[1][:1].to(dev)
    post = LandmarkPostprocessor(Identity(**O.make_identity(0, 37)), device=dev)
    p = O.MAY
    params = StageParams(p["Feat_smooth_sigma"], p["AMP_method"], p["Feat_AMPs"], p["rot_AMP"], p["trans_AMP"],
                         p["Head_smooth_sigma"], p["shoulder_AMP"])
    rng = np.random.default_rng(0)
    pcm = rng.integers(-8000, 8000, size=(800 * n_pushes, 2), dtype=np.int16)
    f32 = (0.2 * rng.standard_normal(267 * n_pushes)).astype(np.float32)
    rs = Resampler(48000, 2, device=dev)

    def session(resampler):
        torch.manual_seed(0)
        return PortraitStream(AudioStream(mel, apc, mouth, head, projector=proj, k=10, percent=1.0, sigma_scale=0.3,
                                          resampler=resampler), post, params, net, cand, size=(512, 512))
    out = {}
    for rnd in range(2):                                  # round 0 warms up
        native, plain = session(rs), session(None)
        t48, t16 = [], []
        for j in range(n_pushes):
            for s, feed, step, times in ((native, pcm, 800, t48), (plain, f32, 267, t16)):
                t0 = time.perf_counter()
                s.push(feed[j * step:(j + 1) * step])
                torch.cuda.synchronize()
                times.append(time.perf_counter() - t0)
        if rnd:
            for key, times in (("pcm16_stereo_48k", t48), ("fp32_16k", t16)):
                ms = np.array(times[100:]) * 1e3              # after the look-ahead's first frame
                out[key] = {"median_ms": float(np.median(ms)), "p99_ms": float(np.percentile(ms, 99)), "n": int(ms.size)}
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--host", action="store_true")
    ap.add_argument("--pushes", type=int, default=700)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    name, limit = card()
    rng = np.random.default_rng(1)
    kernels = {}
    for orig_sr in (44100, 48000):
        for label, ch, dtype in (("fp32_mono", 1, torch.float32), ("pcm16_stereo", 2, torch.int16)):
            rs = Resampler(orig_sr, ch, "kaiser_best", device=dev)
            for clip, seconds in (("11.5s", CLIP_S), ("10min", 600.0)):
                n = int(seconds * orig_sr)
                shape = (n,) if ch == 1 else (n, ch)
                x = torch.from_numpy(rng.integers(-8000, 8000, size=shape, dtype=np.int16)).to(dev)
                x = x if dtype == torch.int16 else (x.float() / 32768.0)
                n_out = rs.n_out(n)
                ms = kernel_ms(rs, x, n_out)
                tp = taps(rs, n)
                kernels[f"{orig_sr}_{label}_{clip}"] = {"outputs": n_out, "kernel_ms": ms, "taps": tp,
                                                        "gtaps_per_s": tp / ms / 1e6}
    res = {"card": name, "power_limit": limit, "filter": "kaiser_best", "kernel": kernels,
           "push": live_pushes(dev, a.pushes)}
    if a.host:
        x = rng.integers(-8000, 8000, size=int(CLIP_S * 48000), dtype=np.int16)
        t0 = time.perf_counter()
        RO.resample(x, 48000, "kaiser_best")
        res["host_numpy_restatement_48k_11.5s_s"] = time.perf_counter() - t0
        res["host_cores"] = os.cpu_count()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
