"""Whole clips (video.render_to_mjpeg) and live streams (video.PortraitRecorder) into Motion-JPEG AVI files: the frames in
the file are the oracle's JPEG bytes of the frames the generator renders, the audio chunks are the samples given, and a
recorded push makes no host synchronisation and keeps device memory flat."""
import io
import os

import numpy as np
import pytest
import torch

import avi_reader
from oracle import jpeg_oracle as J
from oracle import landmark_oracle as O
from test_gpu_landmarks import _params
from test_gpu_portrait_stream import SIZE, _net, _post_of
from test_gpu_stream import _golden as _mel_golden
from test_gpu_stream import _pieces, _stages

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


def _pil(img):
    try:
        from PIL import Image
    except ImportError:
        return None
    b = io.BytesIO()
    Image.fromarray(img).save(b, "JPEG", quality=75)
    return b.getvalue()


def test_render_to_mjpeg_writes_the_oracle_bytes_and_the_audio(tmp_path):
    from livespeechportraits_b200.video import render_to_mjpeg
    from oracle import raster_oracle as R
    net, cand = _net()
    n, batch = 11, 4
    lm, sh = R.make_landmarks(n, (SIZE, SIZE), seed=8, spill=0.1)
    audio = np.random.default_rng(3).standard_normal(16000).astype(np.float32)
    path, fpath, fdir = str(tmp_path / "clip.avi"), str(tmp_path / "maps.avi"), tmp_path / "frames"
    fdir.mkdir()
    info = render_to_mjpeg(net, lm, sh, cand, path, size=(SIZE, SIZE), batch=batch, audio=audio,
                           feature_maps_path=fpath, frames_dir=str(fdir))
    assert info["frames"] == n
    maps = net.draw_feature_maps(torch.from_numpy(lm).to(DEV), torch.from_numpy(sh).to(DEV), (SIZE, SIZE))
    frames = torch.cat([net.render_image(maps[o:o + batch], cand) for o in range(0, n, batch)]).cpu().numpy()
    masks = (maps[:, 0] * 255.0).to(torch.uint8).cpu().numpy()
    want = [J.encode(f, 75) for f in frames]
    want_maps = [J.encode(m, 75) for m in masks]
    r = avi_reader.read(path)
    assert r["data"](b"00dc") == want
    assert b"".join(r["data"](b"01wb")) == audio[:n * 16000 // 60].tobytes()
    assert avi_reader.read(fpath)["data"](b"00dc") == want_maps
    for j in range(n):
        assert (fdir / f"pred_{j + 1}.jpg").read_bytes() == want[j]
        assert (fdir / f"input_{j + 1}.jpg").read_bytes() == want_maps[j]
        for img, name in ((frames[j], "pred"), (masks[j], "input")):
            pil = _pil(img)
            assert pil is None or pil == (fdir / f"{name}_{j + 1}.jpg").read_bytes()
    import cv2
    cap = cv2.VideoCapture(path)
    assert cap.get(cv2.CAP_PROP_FRAME_COUNT) == n and cap.get(cv2.CAP_PROP_FPS) == 60
    assert (cap.get(cv2.CAP_PROP_FRAME_WIDTH), cap.get(cv2.CAP_PROP_FRAME_HEIGHT)) == (SIZE, SIZE)


def _recorder(path, seed=0, projector=True):
    from livespeechportraits_b200.stream import AudioStream, PortraitStream
    from livespeechportraits_b200.video import PortraitRecorder
    mel, apc, mouth, head, proj = _stages()
    net, cand = _net()
    torch.manual_seed(seed)
    a = AudioStream(mel, apc, mouth, head, projector=proj if projector else None, k=10, percent=1.0, sigma_scale=0.3)
    ps = PortraitStream(a, _post_of(O.make_identity(0, 37)), _params(O.MAY), net, cand, size=(SIZE, SIZE))
    return PortraitRecorder(ps, path)


@pytest.mark.parametrize("how", [267, 1600, "random"])
def test_recorder_writes_the_streams_frames_whatever_the_push_sizes(tmp_path, how):
    audio = _mel_golden("mel_00083_wav")["audio"]
    path = str(tmp_path / "live.avi")
    rec = _recorder(path, seed=7)
    frames, at = [], 0
    for k in _pieces(audio.shape[0], how, seed=11):
        frames.append(rec.push(audio[at:at + k]).frames)
        at += k
    frames.append(rec.finish().frames)
    frames = torch.cat(frames).cpu().numpy()
    r = avi_reader.read(path)
    assert r["data"](b"00dc") == [J.encode(f, 75) for f in frames]
    keep = len(frames) * 16000 // 60
    assert b"".join(r["data"](b"01wb")) == audio[:keep].astype(np.float32).tobytes()


def test_recorded_push_makes_no_synchronising_call(tmp_path):
    audio = _mel_golden("mel_00083_wav")["audio"]
    rec = _recorder(str(tmp_path / "sync.avi"))
    at = 0
    while rec.stream.frames < 3:
        rec.push(audio[at:at + 267])
        at += 267
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        r = rec.push(audio[at:at + 267])
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert r.frames.shape[0] == 1
    rec.finish()


def test_recorder_memory_is_flat_over_two_minutes(tmp_path):
    from oracle import mel_oracle as W
    audio = W.make_audio(16000 * 120, seed=5)
    path = str(tmp_path / "long.avi")
    rec = _recorder(path, seed=2, projector=False)
    seen = {}
    for j in range(120):
        rec.push(audio[16000 * j:16000 * (j + 1)])
        seen[j] = torch.cuda.memory_allocated(DEV)
    rec.finish()
    assert seen[9] == seen[119], (seen[9], seen[119])
    r = avi_reader.read(path)
    assert len(r["data"](b"00dc")) == rec.stream.frames > 7000
    assert os.path.getsize(path) == sum(size for _, _, size in r["segments"])
