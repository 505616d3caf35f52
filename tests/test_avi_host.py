"""video.MjpegAviWriter on the host: files built from known JPEG bytes and known audio, read back by cv2 and by the
independent RIFF reader in avi_reader.py."""
import io
import os

import numpy as np
import pytest

import avi_reader
from livespeechportraits_b200.video import MjpegAviWriter
from oracle import jpeg_oracle as J

cv2 = pytest.importorskip("cv2")


def _frames(n, h=64, w=48, seed=0, noise=16):
    """Flat frames of distinct colours plus noise in one corner: decodable to near their colour, so order is visible."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        a = np.empty((h, w, 3), np.uint8)
        a[:] = ((37 * i) % 256, (91 * i + 50) % 256, (13 * i + 200) % 256)
        a[:noise, :noise] = rng.integers(0, 256, (noise, noise, 3))
        out.append(a)
    return out


def _jpeg(a):
    try:
        from PIL import Image
    except ImportError:
        return J.encode(a, 75)
    b = io.BytesIO()
    Image.fromarray(a).save(b, "JPEG", quality=75)
    return b.getvalue()


def _write(path, jpegs, audio, rate, channels, fmt, segment_bytes=1 << 30, pieces=7):
    w = MjpegAviWriter(path, (48, 64), fps=60, audio_rate=rate, audio_channels=channels, audio_format=fmt,
                       segment_bytes=segment_bytes)
    cuts = np.linspace(0, len(audio), pieces + 1).astype(int) if audio is not None else None
    for i, j in enumerate(jpegs):
        if audio is not None and i < pieces:
            w.write_audio(audio[cuts[i]:cuts[i + 1]])
        w.write_frame(j)
    w.close()
    return w


def _check_cv2(path, frames, jpegs):
    cap = cv2.VideoCapture(path)
    assert cap.isOpened()
    assert cap.get(cv2.CAP_PROP_FPS) == 60
    assert (cap.get(cv2.CAP_PROP_FRAME_WIDTH), cap.get(cv2.CAP_PROP_FRAME_HEIGHT)) == (48, 64)
    n = 0
    while True:
        ok, f = cap.read()
        if not ok:
            break
        want = cv2.imdecode(np.frombuffer(jpegs[n], np.uint8), cv2.IMREAD_COLOR)
        # ffmpeg's MJPEG decoder and its YUV->BGR conversion are not libjpeg's, so decoded pixels are close, not equal;
        # the flat colour of each frame identifies it
        assert np.abs(f[32:, 24:].astype(int) - want[32:, 24:]).mean() < 3, n
        n += 1
    assert n == len(frames)


@pytest.mark.parametrize("rate,channels,fmt", [(16000, 1, "f32"), (48000, 2, "s16")])
def test_file_reads_back_with_its_frames_and_audio(tmp_path, rate, channels, fmt):
    frames = _frames(30)
    jpegs = [_jpeg(a) for a in frames]
    rng = np.random.default_rng(1)
    n_audio = rate                                           # 1 s of audio for 0.5 s of video: cut on close
    audio = rng.standard_normal((n_audio, channels)).astype(np.float32) if fmt == "f32" else \
        rng.integers(-32768, 32768, (n_audio, channels), dtype=np.int16)
    if channels == 1:
        audio = audio[:, 0]
    path = str(tmp_path / "clip.avi")
    _write(path, jpegs, audio, rate, channels, fmt)
    _check_cv2(path, frames, jpegs)
    r = avi_reader.read(path)
    assert [s[0] for s in r["strh"]] == [b"vids", b"auds"] and r["strh"][0][1] == b"MJPG"
    assert r["strh"][0][6:8] == (1, 60) and r["strh"][0][9] == 30                       # scale, rate; length
    tag, ch, sr, bps, align, bits = __import__("struct").unpack_from("<HHIIHH", r["strf"][1])
    assert (tag, ch, sr, align, bits) == ((3, channels, rate, 4 * channels, 32) if fmt == "f32" else
                                          (1, channels, rate, 2 * channels, 16))
    assert r["data"](b"00dc") == jpegs
    keep = 30 * rate // 60
    assert b"".join(r["data"](b"01wb")) == np.ascontiguousarray(audio[:keep]).tobytes()
    assert r["strh"][1][9] == keep
    assert len(r["idx1"]) == len(r["movi_chunks"])
    # interleaving: every audio chunk follows the frame during which it starts
    order = [c for c, _, _ in r["movi_chunks"]]
    assert order[0] == b"00dc"
    at, frame = 0, 0
    for c, _, size in r["movi_chunks"]:
        if c == b"00dc":
            frame += 1
        else:
            assert (frame - 1) * rate // 60 <= at < frame * rate // 60
            at += size // (audio.itemsize * channels)


def test_segments_past_the_limit_become_avix(tmp_path):
    frames = _frames(300, seed=3, noise=32)
    jpegs = [_jpeg(a) for a in frames]
    audio = np.random.default_rng(2).standard_normal(16000 * 6).astype(np.float32)
    path = str(tmp_path / "long.avi")
    _write(path, jpegs, audio, 16000, 1, "f32", segment_bytes=256 << 10, pieces=300)
    r = avi_reader.read(path)
    forms = [f for f, _, _ in r["segments"]]
    assert forms[0] == b"AVI " and forms.count(b"AVIX") >= 2
    assert all(size <= (256 << 10) + 4096 for _, _, size in r["segments"])
    assert r["data"](b"00dc") == jpegs
    assert b"".join(r["data"](b"01wb")) == audio[:300 * 16000 // 60].tobytes()
    vid = dict(r["odml"])[b"00dc"]
    assert vid == [at for c, at, _ in r["movi_chunks"] if c == b"00dc"]
    _check_cv2(path, frames, jpegs)


def test_zero_frame_file_is_valid(tmp_path):
    path = str(tmp_path / "empty.avi")
    w = MjpegAviWriter(path, (48, 64), audio_rate=16000)
    w.write_audio(np.zeros(1000, np.float32))
    w.close()
    r = avi_reader.read(path)
    assert r["movi_chunks"] == [] and r["idx1"] == [] and r["strh"][0][9] == 0 and r["strh"][1][9] == 0
    assert os.path.getsize(path) == r["segments"][0][2]


def test_bad_arguments_are_refused(tmp_path):
    with pytest.raises(ValueError, match="audio_format"):
        MjpegAviWriter(str(tmp_path / "a.avi"), (16, 16), audio_format="u8")
    w = MjpegAviWriter(str(tmp_path / "b.avi"), (16, 16), audio_rate=16000)
    with pytest.raises(ValueError, match="float32"):
        w.write_audio(np.zeros(4, np.int16))
    w.close()
