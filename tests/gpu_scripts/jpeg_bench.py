"""Time the GPU JPEG encoder (include/lspj.h) and the Motion-JPEG paths built on it.

    python tests/gpu_scripts/jpeg_bench.py [--frames 672,10000]

Prints ONE JSON line with:
  * the encoder's kernel time per frame at 512 x 512, quality 75, batch 1 and 32, RGB and grey, on the ``large``
    generator's own frames (and masks) and on uniform noise (the worst case for the entropy coder): CUDA events around
    200 ``encode_into`` calls after a warm-up; plus the split over its four kernels from a torch.profiler run;
  * whole clips of each ``--frames`` length from landmark tracks: ``ClipRenderer.render_clip_from_landmarks`` with uint8
    output alone, ``video.render_to_mjpeg`` (quality 75, batch 32) and ``video.render_to_video`` (cv2 DIVX), wall time;
  * a live ``PortraitStream`` at 512 x 512 in one-video-frame pushes (267 samples), with and without a
    ``PortraitRecorder``: median and p99 of the host clock around ``push`` + ``torch.cuda.synchronize()``.
Card name and power limit come from a read-only nvidia-smi query in the same run.  Temporary files go to a temporary
directory that is removed.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
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
from livespeechportraits_b200.jpeg import JpegEncoder  # noqa: E402
from livespeechportraits_b200.landmarks import Identity, LandmarkPostprocessor, StageParams  # noqa: E402
from livespeechportraits_b200.manifold import ManifoldProjector  # noqa: E402
from livespeechportraits_b200.pipeline import ClipRenderer  # noqa: E402
from livespeechportraits_b200.recurrent import ApcEncoder, MouthGenerator  # noqa: E402
from livespeechportraits_b200.stream import AudioStream, PortraitStream  # noqa: E402
from livespeechportraits_b200.video import PortraitRecorder, render_to_mjpeg, render_to_video  # noqa: E402
from oracle import a2h_oracle as A  # noqa: E402
from oracle import f2f_oracle as F  # noqa: E402
from oracle import landmark_oracle as O  # noqa: E402
from oracle import lle_oracle as M  # noqa: E402
from oracle import raster_oracle as RO  # noqa: E402
from oracle import rnn_oracle as R  # noqa: E402

S = 512


def encoder_us(enc, imgs, iters=200):
    n, h, w = imgs.shape[:3]
    c = 3 if imgs.dim() == 4 else 1
    out = torch.empty((n, enc.max_bytes(h, w, c)), dtype=torch.uint8, device=imgs.device)
    sizes = torch.empty(n, dtype=torch.int32, device=imgs.device)
    ws = torch.empty(enc.workspace_bytes(n, h, w, c), dtype=torch.uint8, device=imgs.device)
    for _ in range(10):
        enc.encode_into(imgs, out, sizes, ws)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        enc.encode_into(imgs, out, sizes, ws)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters / n, float(sizes.float().mean())


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", default="672,10000")
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    name, limit = card()
    res = {"card": name, "power_limit": limit}
    net = Feature2Face_G(types.SimpleNamespace(isTrain=False, size="large", n_downsample_G=8, ngf=64, fp16=0))
    net.load_state_dict(F.make_state_dict("large", "B"))
    net = net.to(dev).eval()
    _, cand = F.make_inputs(1, S, S, seed=6)
    cand = cand[:1].to(dev)
    lm, sh = RO.make_landmarks(32, (S, S), seed=3)
    maps = net.draw_feature_maps(torch.from_numpy(lm).to(dev), torch.from_numpy(sh).to(dev), (S, S))
    frames = net.render_image(maps, cand)
    masks = (maps[:, 0] * 255.0).to(torch.uint8)
    noise = torch.randint(0, 256, (32, S, S, 3), dtype=torch.uint8, device=dev)
    enc = JpegEncoder(dev, 75)
    timing = {}
    for label, imgs in (("rgb_frames", frames), ("grey_masks", masks), ("rgb_noise", noise), ("grey_noise", noise[..., 0].contiguous())):
        for b in (1, 32):
            us, mean = encoder_us(enc, imgs[:b].contiguous())
            timing[f"{label}_b{b}"] = {"us_per_frame": round(us, 2), "mean_bytes": round(mean)}
    res["encoder_512_q75"] = timing
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(20):
            enc.encode(frames)
        torch.cuda.synchronize()
    split = {}
    for ev in prof.events():
        t = getattr(ev, "device_time", None)
        if t is None:
            t = getattr(ev, "cuda_time", 0.0)
        if "lspj_" in ev.name and t:
            k = ev.name.split("lspj_")[1].split("(")[0].split("<")[0]
            split[k] = split.get(k, 0.0) + t / 20 / 32
    res["encoder_split_us_per_frame_b32_frames"] = {k: round(v, 3) for k, v in split.items()}

    # whole clips
    clips = {}
    with tempfile.TemporaryDirectory() as tmp:
        for n in [int(x) for x in a.frames.split(",")]:
            lmn, shn = RO.make_landmarks(n, (S, S), seed=4)
            audio = np.random.default_rng(0).standard_normal(n * 16000 // 60 + 100).astype(np.float32)
            row = {}
            clip = ClipRenderer(net, batch=32, device=dev, uint8=True)
            host = torch.empty((n, S, S, 3), dtype=torch.uint8).pin_memory()
            lt, st = torch.from_numpy(lmn).pin_memory(), torch.from_numpy(shn).pin_memory()
            clip.render_clip_from_landmarks(lt[:64], st[:64], cand, host[:64], (S, S))     # warm-up
            render_to_mjpeg(net, lmn[:64], shn[:64], cand, os.path.join(tmp, "w.avi"), size=(S, S), audio=audio)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            clip.render_clip_from_landmarks(lt, st, cand, host, (S, S))
            torch.cuda.synchronize()
            row["uint8_render_s"] = round(time.perf_counter() - t0, 3)
            t0 = time.perf_counter()
            info = render_to_mjpeg(net, lmn, shn, cand, os.path.join(tmp, "m.avi"), size=(S, S), audio=audio)
            row["render_to_mjpeg_s"] = round(time.perf_counter() - t0, 3)
            row["mjpeg_writer_busy_s"] = round(info["encode_seconds"], 3)
            row["mjpeg_file_mb"] = round(info["bytes"] / 1e6, 1)
            t0 = time.perf_counter()
            vinfo = render_to_video(net, lmn, shn, cand, os.path.join(tmp, "d.avi"), size=(S, S))
            row["render_to_video_divx_s"] = round(time.perf_counter() - t0, 3)
            row["divx_writer_busy_s"] = round(vinfo["encode_seconds"], 3)
            clips[str(n)] = row
    res["clips_512"] = clips

    # live
    g = np.load(os.path.join(ROOT, "tests", "golden", "mel", "mel_00083_wav.npz"))
    audio = g["audio"]
    mopt, hopt = R.default_mouth_opt(), A.default_opt()
    mel, apc = MelFrontEnd(g["basis"], device=dev), ApcEncoder(R.make_apc_state_dict("B", 0), device=dev)
    mouth = MouthGenerator(mopt, R.make_mouth_state_dict(mopt, "B", 0), device=dev)
    head = HeadposeGenerator(hopt, A.make_state_dict(hopt, "B", 1), device=dev)
    proj = ManifoldProjector(M.make_database(10_000, 512, seed=1), device=dev)
    post = LandmarkPostprocessor(Identity(**O.make_identity(0, 37)), device=dev)
    p = O.MAY
    params = StageParams(p["Feat_smooth_sigma"], p["AMP_method"], p["Feat_AMPs"], p["rot_AMP"], p["trans_AMP"],
                         p["Head_smooth_sigma"], p["shoulder_AMP"])
    live = {}
    with tempfile.TemporaryDirectory() as tmp:
        for rep in range(2):                                   # the first round warms up
            for record in (False, True):
                torch.manual_seed(0)
                s = PortraitStream(AudioStream(mel, apc, mouth, head, projector=proj, k=10, percent=1.0,
                                               sigma_scale=0.3), post, params, net, cand, size=(S, S))
                r = PortraitRecorder(s, os.path.join(tmp, f"l{rep}.avi")) if record else s
                times = []
                for at in range(0, audio.shape[0], 267):
                    t0 = time.perf_counter()
                    out = r.push(audio[at:at + 267])
                    torch.cuda.synchronize()
                    if out.frames.shape[0]:
                        times.append(time.perf_counter() - t0)
                r.finish()
                torch.cuda.synchronize()
                ms = np.array(times) * 1e3
                if rep:
                    live["recorded" if record else "plain"] = {"median_ms": round(float(np.median(ms)), 3),
                                                               "p99_ms": round(float(np.percentile(ms, 99)), 3),
                                                               "pushes": len(ms)}
    res["live_push_512"] = live
    print(json.dumps(res))


if __name__ == "__main__":
    main()
