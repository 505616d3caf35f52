"""Whole clips (video.render_to_h264) and live streams (video.PortraitRecorder(codec="h264")) into H.264 AVI files: the
video chunks concatenate to the encoder's stream of the rendered frames, keyframe flags sit exactly on the IDRs, the
audio is what render_to_mjpeg writes for the same clip, and a recorded session is the whole-clip encode of its frames."""
import numpy as np
import pytest
import torch

import avi_reader
from livespeechportraits_b200.h264 import H264Encoder
from oracle import h264_oracle as H
from oracle import landmark_oracle as O
from test_gpu_landmarks import _params
from test_gpu_portrait_stream import SIZE, _net, _post_of
from test_gpu_stream import _golden as _mel_golden
from test_gpu_stream import _pieces, _stages

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


def test_render_to_h264_writes_the_encoders_stream_and_the_audio(tmp_path):
    from livespeechportraits_b200.video import render_to_h264, render_to_mjpeg
    from oracle import raster_oracle as R
    net, cand = _net()
    n, batch = 11, 4
    lm, sh = R.make_landmarks(n, (SIZE, SIZE), seed=8, spill=0.1)
    audio = np.random.default_rng(3).standard_normal(16000).astype(np.float32)
    path, fpath, mpath = str(tmp_path / "clip.avi"), str(tmp_path / "maps.avi"), str(tmp_path / "clip_mjpeg.avi")
    info = render_to_h264(net, lm, sh, cand, path, size=(SIZE, SIZE), batch=batch, qp=26, gop=5, audio=audio,
                          feature_maps_path=fpath)
    assert info["frames"] == n
    render_to_mjpeg(net, lm, sh, cand, mpath, size=(SIZE, SIZE), batch=batch, audio=audio)
    maps = net.draw_feature_maps(torch.from_numpy(lm).to(DEV), torch.from_numpy(sh).to(DEV), (SIZE, SIZE))
    frames = torch.cat([net.render_image(maps[o:o + batch], cand) for o in range(0, n, batch)])
    masks = (maps[:, 0] * 255.0).to(torch.uint8)
    enc = H264Encoder(DEV, qp=26, gop=5)
    want = enc.encode(frames).to_bytes()
    assert want == H.encode(frames.cpu().numpy(), qp=26, gop=5)[0]
    r = avi_reader.read(path)
    assert r["strh"][0][1] == b"H264"
    assert r["data"](b"00dc") == want
    assert [bool(flags & 0x10) for cid, flags, _, _ in r["idx1"] if cid == b"00dc"] == [i % 5 == 0 for i in range(n)]
    assert r["data"](b"01wb") == avi_reader.read(mpath)["data"](b"01wb")
    assert b"".join(r["data"](b"01wb")) == audio[:n * 16000 // 60].tobytes()
    assert avi_reader.read(fpath)["data"](b"00dc") == enc.encode(masks).to_bytes()
    import cv2
    cap = cv2.VideoCapture(path)
    got = 0
    while cap.read()[0]:
        got += 1
    assert got == n


def _recorder(path, codec, seed=0):
    from livespeechportraits_b200.stream import AudioStream, PortraitStream
    from livespeechportraits_b200.video import PortraitRecorder
    mel, apc, mouth, head, proj = _stages()
    net, cand = _net()
    torch.manual_seed(seed)
    a = AudioStream(mel, apc, mouth, head, projector=proj, k=10, percent=1.0, sigma_scale=0.3)
    ps = PortraitStream(a, _post_of(O.make_identity(0, 37)), _params(O.MAY), net, cand, size=(SIZE, SIZE))
    return PortraitRecorder(ps, path, codec=codec, qp=28, gop=8)


@pytest.mark.parametrize("how", [267, "random"])
def test_recorder_records_the_whole_clip_stream_of_its_frames(tmp_path, how):
    audio = _mel_golden("mel_00083_wav")["audio"]
    path = str(tmp_path / "live.avi")
    rec = _recorder(path, "h264", seed=7)
    frames, at = [], 0
    for k in _pieces(audio.shape[0], how, seed=11):
        frames.append(rec.push(audio[at:at + k]).frames)
        at += k
    frames.append(rec.finish().frames)
    frames = torch.cat(frames)
    r = avi_reader.read(path)
    assert r["data"](b"00dc") == H264Encoder(DEV, qp=28, gop=8).encode(frames).to_bytes()
    assert [bool(flags & 0x10) for cid, flags, _, _ in r["idx1"] if cid == b"00dc"] == \
        [i % 8 == 0 for i in range(frames.shape[0])]
    keep = len(frames) * 16000 // 60
    assert b"".join(r["data"](b"01wb")) == audio[:keep].astype(np.float32).tobytes()


def test_recorded_h264_push_makes_no_synchronising_call(tmp_path):
    audio = _mel_golden("mel_00083_wav")["audio"]
    rec = _recorder(str(tmp_path / "sync.avi"), "h264")
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
