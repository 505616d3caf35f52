"""Time the GPU H.264 encoder (include/lspv.h) and measure what it stores, next to the JPEG encoder.

    python tests/gpu_scripts/h264_bench.py

Prints ONE JSON line with:
  * encode time per frame at 512 x 512 on the ``large`` generator's frames, from CUDA events: batch 1 (one call per
    frame, 200 calls after a warm-up) for an I frame (gop 1) and a P frame, and a 672-frame clip in one call, all I
    (gop 1), all P but the first, and gop 60; plus the split over the kernels of the gop-60 clip from a torch.profiler run;
  * bytes per frame and Y PSNR against the source's Y (the BT.601 formula of lspv.h) at QP 20, 26 and 32 (gop 60) for
    a 672-frame talking-head clip - the frames a live PortraitStream renders from the golden speech clip - next to
    ``JpegEncoder`` at quality 75 (its files decoded by cv2.imdecode, the H.264 stream by opencv-python's libavcodec);
  * a live ``PortraitStream`` at 512 x 512 in one-video-frame pushes (267 samples) with an MJPEG and an H.264
    ``PortraitRecorder``: median and p99 of the host clock around ``push`` + ``torch.cuda.synchronize()``.
Card name and power limit come from a read-only nvidia-smi query in the same run.  Temporary files go to a temporary
directory that is removed.
"""
from __future__ import annotations

import json
import os
import sys
import tempfile
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import libavcodec  # noqa: E402
from lle_bench import card  # noqa: E402
from livespeechportraits_b200.audio import MelFrontEnd  # noqa: E402
from livespeechportraits_b200.generator import Feature2Face_G  # noqa: E402
from livespeechportraits_b200.h264 import H264Encoder  # noqa: E402
from livespeechportraits_b200.headpose import HeadposeGenerator  # noqa: E402
from livespeechportraits_b200.jpeg import JpegEncoder  # noqa: E402
from livespeechportraits_b200.landmarks import Identity, LandmarkPostprocessor, StageParams  # noqa: E402
from livespeechportraits_b200.manifold import ManifoldProjector  # noqa: E402
from livespeechportraits_b200.recurrent import ApcEncoder, MouthGenerator  # noqa: E402
from livespeechportraits_b200.stream import AudioStream, PortraitStream  # noqa: E402
from livespeechportraits_b200.video import PortraitRecorder  # noqa: E402
from oracle import a2h_oracle as A  # noqa: E402
from oracle import f2f_oracle as F  # noqa: E402
from oracle import h264_oracle as HO  # noqa: E402
from oracle import landmark_oracle as O  # noqa: E402
from oracle import lle_oracle as M  # noqa: E402
from oracle import raster_oracle as RO  # noqa: E402
from oracle import rnn_oracle as R  # noqa: E402

S = 512
CLIP = 672


def timed(fn, iters):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def encoder_times(dev, frames):
    """Encode time per frame (us): batch 1 I and P, and one 672-frame call at gop 1, all-P and gop 60."""
    out = {}
    h, w = frames.shape[1:3]
    for label, gop in (("I_b1", 1), ("P_b1", 1 << 30)):
        enc = H264Encoder(dev, qp=26, gop=gop)
        state = enc.new_state(h, w)
        data = torch.empty((1, enc.max_bytes(h, w)), dtype=torch.uint8, device=dev)
        sizes = torch.empty(1, dtype=torch.int32, device=dev)
        idr = torch.empty(1, dtype=torch.uint8, device=dev)
        ws = enc.workspace(h, w)
        enc.encode_into(frames[:1], 0, state, data, sizes, idr, ws)
        k = [0]

        def one():
            k[0] += 1
            enc.encode_into(frames[k[0] % frames.shape[0]:][:1], 1, state, data, sizes, idr, ws)
        out[label] = {"us_per_frame": round(1e3 * timed(one, 200), 1)}
    n = frames.shape[0]
    for label, gop in (("I_clip", 1), ("P_clip", 1 << 30), ("gop60_clip", 60)):
        enc = H264Encoder(dev, qp=26, gop=gop)
        state = enc.new_state(h, w)
        data = torch.empty((n, enc.max_bytes(h, w)), dtype=torch.uint8, device=dev)
        sizes = torch.empty(n, dtype=torch.int32, device=dev)
        idr = torch.empty(n, dtype=torch.uint8, device=dev)
        ws = enc.workspace(h, w)
        ms = timed(lambda: enc.encode_into(frames, 0, state, data, sizes, idr, ws), 3)
        out[label] = {"us_per_frame": round(1e3 * ms / n, 1), "frames": n}
    from torch.profiler import ProfilerActivity, profile
    enc = H264Encoder(dev, qp=26, gop=60)
    enc.encode(frames)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        enc.encode(frames)
        torch.cuda.synchronize()
    split = {}
    for ev in prof.events():
        t = getattr(ev, "device_time", None)
        if t is None:
            t = getattr(ev, "cuda_time", 0.0)
        if "lspv_" in ev.name and t:
            key = ev.name.split("lspv_")[1].split("(")[0].split("<")[0]
            split[key] = split.get(key, 0.0) + t / n
    out["gop60_clip_split_us_per_frame"] = {k: round(v, 2) for k, v in split.items()}
    return out


def psnr(a, b):
    mse = float(np.mean((a.astype(np.float64) - b) ** 2))
    return 99.0 if mse == 0 else 10 * np.log10(255.0 ** 2 / mse)


def sizes_and_quality(dev, frames):
    import cv2
    src_y = [HO.to_yuv(f)[0] for f in frames.cpu().numpy()]
    out = {}
    for qp in (20, 26, 32):
        aus = H264Encoder(dev, qp=qp, gop=60).encode(frames).to_bytes()
        dec = libavcodec.decode(aus)
        idr = [i % 60 == 0 for i in range(len(aus))]
        out[f"h264_qp{qp}"] = {
            "bytes_per_frame": round(sum(map(len, aus)) / len(aus)),
            "bytes_per_I": round(np.mean([len(a) for a, k in zip(aus, idr) if k])),
            "bytes_per_P": round(np.mean([len(a) for a, k in zip(aus, idr) if not k])),
            "y_psnr_db": round(float(np.mean([psnr(d[0], y) for d, y in zip(dec, src_y)])), 2)}
    files = JpegEncoder(dev, 75).encode(frames).to_bytes()
    ys = [HO.to_yuv(cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR)[:, :, ::-1])[0] for f in files]
    out["jpeg_q75"] = {"bytes_per_frame": round(sum(map(len, files)) / len(files)),
                       "y_psnr_db": round(float(np.mean([psnr(d, y) for d, y in zip(ys, src_y)])), 2)}
    return out


def stages(dev):
    g = np.load(os.path.join(ROOT, "tests", "golden", "mel", "mel_00083_wav.npz"))
    mopt, hopt = R.default_mouth_opt(), A.default_opt()
    mel, apc = MelFrontEnd(g["basis"], device=dev), ApcEncoder(R.make_apc_state_dict("B", 0), device=dev)
    mouth = MouthGenerator(mopt, R.make_mouth_state_dict(mopt, "B", 0), device=dev)
    head = HeadposeGenerator(hopt, A.make_state_dict(hopt, "B", 1), device=dev)
    proj = ManifoldProjector(M.make_database(10_000, 512, seed=1), device=dev)
    post = LandmarkPostprocessor(Identity(**O.make_identity(0, 37)), device=dev)
    p = O.MAY
    params = StageParams(p["Feat_smooth_sigma"], p["AMP_method"], p["Feat_AMPs"], p["rot_AMP"], p["trans_AMP"],
                         p["Head_smooth_sigma"], p["shoulder_AMP"])
    return g["audio"], (mel, apc, mouth, head, proj, post, params)


def main() -> None:
    dev = torch.device("cuda", 0)
    name, limit = card()
    res = {"card": name, "power_limit": limit}
    net = Feature2Face_G(types.SimpleNamespace(isTrain=False, size="large", n_downsample_G=8, ngf=64, fp16=0))
    net.load_state_dict(F.make_state_dict("large", "B"))
    net = net.to(dev).eval()
    _, cand = F.make_inputs(1, S, S, seed=6)
    cand = cand[:1].to(dev)
    audio, (mel, apc, mouth, head, proj, post, params) = stages(dev)

    def portrait():
        torch.manual_seed(0)
        return PortraitStream(AudioStream(mel, apc, mouth, head, projector=proj, k=10, percent=1.0, sigma_scale=0.3),
                              post, params, net, cand, size=(S, S))

    # the talking-head clip: what a live stream renders from the golden speech clip
    s = portrait()
    frames = [s.push(audio).frames, s.finish().frames]
    talking = torch.cat(frames)[:CLIP].contiguous()
    res["talking_head_frames"] = int(talking.shape[0])
    lm, sh = RO.make_landmarks(32, (S, S), seed=3)
    maps = net.draw_feature_maps(torch.from_numpy(lm).to(dev), torch.from_numpy(sh).to(dev), (S, S))
    res["encode_512_qp26"] = encoder_times(dev, talking)
    res["encode_512_qp26_jittered_landmarks_b1"] = encoder_times(dev, net.render_image(maps, cand))["P_b1"]
    res["size_quality_512"] = sizes_and_quality(dev, talking)

    live = {}
    with tempfile.TemporaryDirectory() as tmp:
        for rep in range(2):                                   # the first round warms up
            for codec in ("mjpeg", "h264"):
                r = PortraitRecorder(portrait(), os.path.join(tmp, f"l{rep}{codec}.avi"), codec=codec)
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
                    live[codec] = {"median_ms": round(float(np.median(ms)), 3),
                                   "p99_ms": round(float(np.percentile(ms, 99)), 3), "pushes": len(ms),
                                   "file_bytes": os.path.getsize(os.path.join(tmp, f"l{rep}{codec}.avi"))}
    res["live_push_512_recorded"] = live
    print(json.dumps(res))


if __name__ == "__main__":
    main()
