"""Clip -> video file: the body of the reference's render loop without its JPEG round trip (SURVEY.md 8f, row N3).

The reference renders one frame per iteration (demo.py:260-266), converts it with ``util.tensor2im`` (demo.py:268),
writes it as a JPEG (``visualizer.save_images``, util/visualizer.py:120-143), later re-reads every JPEG with
``cv2.imread`` and pushes it into ``cv2.VideoWriter('DIVX', 60 fps)`` (demo.py:35-45), muxes the audio with ffmpeg
(demo.py:43-44) and deletes the JPEGs (demo.py:286-289).  Here the landmark tracks of the whole clip go to the GPU once,
batches are rasterised + rendered + converted to uint8 HWC images by the generator's kernels
(``ClipRenderer.render_clip_from_landmarks``), and a writer thread feeds the frames of each batch to ONE
``cv2.VideoWriter`` as they land in pinned host memory, while the next batches render.  Same container / codec / fps
as the reference; the frames do not pass through a lossy JPEG first.
"""
from __future__ import annotations

import os
import queue
import shutil
import struct
import subprocess
import threading
import time
from typing import List, Optional

import numpy as np
import torch

from . import _lib
from .pipeline import ClipRenderer


def _open_writer(path: str, fps: float, size: tuple, fourcc: str):
    import cv2
    w = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*fourcc), fps, (int(size[0]), int(size[1])))
    if not w.isOpened():
        raise RuntimeError(f"cv2.VideoWriter could not open {path!r} with fourcc {fourcc!r}")
    return w


class _WriterThread:
    """Consumes (RGB uint8 [n,H,W,3]) batches in order and writes them as BGR frames; one encoder, one thread."""

    def __init__(self, writer):
        self.writer = writer
        self.q: "queue.Queue" = queue.Queue()
        self.error: Optional[BaseException] = None
        self.busy_seconds = 0.0
        self.frames = 0
        self.thread = threading.Thread(target=self._run, daemon=True)
        self.thread.start()

    def _run(self):
        import cv2
        try:
            while True:
                item = self.q.get()
                if item is None:
                    return
                t0 = time.perf_counter()
                for frame in item:
                    self.writer.write(cv2.cvtColor(frame, cv2.COLOR_RGB2BGR))     # demo.py:41 writes what cv2.imread returned: BGR
                self.frames += len(item)
                self.busy_seconds += time.perf_counter() - t0
        except BaseException as exc:      # noqa: BLE001 - surfaced by close()
            self.error = exc

    def put(self, frames: np.ndarray) -> None:
        self.q.put(frames)

    def close(self) -> None:
        self.q.put(None)
        self.thread.join()
        self.writer.release()
        if self.error is not None:
            raise self.error


def mux_audio(video_path: str, audio_path: str, output_path: str) -> bool:
    """demo.py:43-44: ``ffmpeg -i video -i audio -codec copy -shortest output``.  Returns False when no ffmpeg binary exists."""
    exe = shutil.which("ffmpeg")
    if exe is None:
        return False
    subprocess.check_call([exe, "-y", "-loglevel", "error", "-i", video_path, "-i", audio_path, "-codec", "copy", "-shortest",
                           output_path])
    return True


def _tracks(x, dev):
    """A CUDA tensor stays on the device (fp32, contiguous); numpy goes to pinned host memory for one upload."""
    if isinstance(x, torch.Tensor) and x.is_cuda:
        return x.to(device=dev, dtype=torch.float32).contiguous()
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).pin_memory()


def render_to_video(net, landmarks, shoulders, cand_device: torch.Tensor, output_path: str,
                    size: tuple = (512, 512), fps: float = 60.0, batch: int = 32, fourcc: str = "DIVX",
                    audio_path: Optional[str] = None, feature_maps_path: Optional[str] = None,
                    precision: Optional[str] = None) -> dict:
    """Render a clip from its landmark tracks straight into a video file.

    ``landmarks`` [N,73,2] and ``shoulders`` [N,18,2] (or None) are the per-frame tracks demo.py:237-258 computes
    (``pred_landmarks`` / ``pred_shoulders``), as numpy or as CUDA tensors (``LandmarkPostprocessor.run``'s output, used
    without a host round trip); ``cand_device`` is ``img_candidates`` (demo.py:95).  ``size`` = (W, H) =
    ``(opt.loadSize, opt.loadSize)``.  ``feature_maps_path``: also write the rasterised input maps as a second video
    (demo.py:282-283, ``save_feature_maps``).  ``audio_path``: mux it like demo.py:43-44 when an ffmpeg binary exists.
    Returns ``{"frames", "seconds", "encode_seconds", "writer", "audio_muxed"}``.
    """
    n = int(landmarks.shape[0])
    w, h = int(size[0]), int(size[1])
    dev = cand_device.device
    lm_tracks = _tracks(landmarks, dev)
    sh_tracks = None if shoulders is None else _tracks(shoulders, dev)
    frames_host = torch.empty((n, h, w, 3), dtype=torch.uint8).pin_memory()
    frames_np = frames_host.numpy()
    want_mux = audio_path is not None and shutil.which("ffmpeg") is not None
    video_path = output_path
    if want_mux:
        root, ext = os.path.splitext(output_path)
        video_path = root + ".noaudio" + ext
    t0 = time.perf_counter()
    wt = _WriterThread(_open_writer(video_path, fps, (w, h), fourcc))
    clip = ClipRenderer(net, batch=batch, device=dev, precision=precision, uint8=True)
    try:
        clip.render_clip_from_landmarks(lm_tracks, sh_tracks, cand_device, frames_host, (w, h),
                                        on_batch=lambda off, ln: wt.put(frames_np[off:off + ln]))
    finally:
        wt.close()
    info = {"frames": n, "encode_seconds": wt.busy_seconds, "writer": f"cv2.VideoWriter {fourcc} {fps:g} fps {w}x{h}",
            "audio_muxed": False}
    if feature_maps_path is not None:
        fw = _WriterThread(_open_writer(feature_maps_path, fps, (w, h), fourcc))
        try:
            lm_dev = lm_tracks.to(dev)
            sh_dev = None if sh_tracks is None else sh_tracks.to(dev)
            for off in range(0, n, batch):
                fm = net.draw_feature_maps(lm_dev[off:off + batch], None if sh_dev is None else sh_dev[off:off + batch], (w, h))
                gray = (fm[:, 0] * 255.0).to(torch.uint8).cpu().numpy()                   # demo.py:270: np.uint8(map * 255)
                fw.put(np.repeat(gray[..., None], 3, axis=3))                             # cv2.imread of a grey JPEG: 3 equal channels
        finally:
            fw.close()
    if want_mux:
        info["audio_muxed"] = mux_audio(video_path, audio_path, output_path)
        if info["audio_muxed"]:
            os.remove(video_path)
        else:
            os.replace(video_path, output_path)
    info["seconds"] = time.perf_counter() - t0
    return info


# ---- Motion-JPEG AVI with audio -----------------------------------------------------------------------------------

_SUPER_ENTRIES = 256                       # OpenDML super-index slots per stream: RIFF segments a file may have
_KEYFRAME = 0x10


class MjpegAviWriter:
    """A Motion-JPEG AVI file (fourcc ``MJPG``) with an optional audio stream, written without ffmpeg.

    ``write_frame(jpeg_bytes)`` appends one complete .jpg file as a frame; ``write_audio(samples)`` appends audio: numpy
    ``[n]`` or ``[n, channels]`` samples, float32 (``audio_format="f32"``, WAVE_FORMAT_IEEE_FLOAT, what demo.py's
    ``write_wav`` + ``ffmpeg -codec copy`` puts in its .avi) or int16 (``"s16"``, PCM).  Audio is written in chunks after
    the frame during which the chunk starts, and ``close()`` cuts it to ``floor(frames * audio_rate / fps)`` samples, as
    demo.py's ``-shortest`` does.  The file has an ``idx1`` index and OpenDML (AVI 2.0) ``indx`` / ``ix##`` indices; a
    RIFF segment that would pass ``segment_bytes`` is closed and the file goes on in ``RIFF AVIX`` segments, so files past
    the 1 GB of AVI 1.0 stay readable."""

    def __init__(self, path: str, size, fps: float = 60, audio_rate: Optional[int] = None, audio_channels: int = 1,
                 audio_format: str = "f32", segment_bytes: int = 1 << 30):
        if audio_format not in ("f32", "s16"):
            raise ValueError(f"audio_format must be 'f32' or 's16' (got {audio_format!r})")
        if audio_channels not in (1, 2):
            raise ValueError(f"audio_channels must be 1 or 2 (got {audio_channels})")
        self.width, self.height = int(size[0]), int(size[1])
        self.fps = float(fps)
        self.audio_rate = None if audio_rate is None else int(audio_rate)
        self.channels = int(audio_channels)
        self.dtype = np.float32 if audio_format == "f32" else np.int16
        self.block_align = self.channels * np.dtype(self.dtype).itemsize
        self.segment_bytes = int(segment_bytes)
        self.frames = 0
        self.samples = 0                   # audio sample frames written to the file
        self._pending: List[np.ndarray] = []
        self._pending_n = 0
        self._f = open(path, "wb")
        self._streams = 1 if self.audio_rate is None else 2
        self._max_chunk = 0
        self._segments: List[list] = [[], []]      # per stream: (ix offset, ix size, duration) of closed segments
        self._idx1: List[tuple] = []
        self._write_header()
        self._open_segment(first=True)

    # -- layout ---------------------------------------------------------------------------------------------------
    def _rate(self):
        if float(self.fps).is_integer():
            return 1, int(self.fps)
        return 1000, int(round(self.fps * 1000))

    def _write_header(self):
        f = self._f
        f.write(b"RIFF\0\0\0\0AVI LIST\0\0\0\0hdrl")
        self._avih = f.tell() + 8
        f.write(b"avih" + struct.pack("<I", 56) + bytes(56))
        self._strh, self._indx = [], []
        for s in range(self._streams):
            strl = f.tell()
            f.write(b"LIST\0\0\0\0strl")
            self._strh.append(f.tell() + 8)
            f.write(b"strh" + struct.pack("<I", 56) + bytes(56))
            if s == 0:
                f.write(b"strf" + struct.pack("<IIiiHH4sIiiII", 40, 40, self.width, self.height, 1, 24, b"MJPG",
                                              self.width * self.height * 3, 0, 0, 0, 0))
            else:
                fmt = 3 if self.dtype == np.float32 else 1
                f.write(b"strf" + struct.pack("<IHHIIHHH", 18, fmt, self.channels, self.audio_rate,
                                              self.audio_rate * self.block_align, self.block_align,
                                              8 * np.dtype(self.dtype).itemsize, 0))
            self._indx.append(f.tell())
            f.write(b"indx" + struct.pack("<I", 24 + 16 * _SUPER_ENTRIES) + bytes(24 + 16 * _SUPER_ENTRIES))
            self._patch_size(strl)
        odml = f.tell()
        f.write(b"LIST\0\0\0\0odml")
        self._dmlh = f.tell() + 8
        f.write(b"dmlh" + struct.pack("<I", 248) + bytes(248))
        self._patch_size(odml)
        self._patch_size(12)

    def _patch_size(self, at: int, end: Optional[int] = None):
        end = self._f.tell() if end is None else end
        self._f.seek(at + 4)
        self._f.write(struct.pack("<I", end - at - 8))
        self._f.seek(end)

    def _open_segment(self, first: bool):
        f = self._f
        if not first:
            self._riff = f.tell()
            f.write(b"RIFF\0\0\0\0AVIX")
        else:
            self._riff = 0
        self._movi = f.tell()
        f.write(b"LIST\0\0\0\0movi")
        self._chunks: List[List[tuple]] = [[], []]     # per stream: (data offset, size, duration)
        self._first = first

    def _close_segment(self):
        f = self._f
        for s in range(self._streams):
            chunks = self._chunks[s]
            if not chunks:
                continue
            at = f.tell()
            base = self._movi
            cid = b"00dc" if s == 0 else b"01wb"
            f.write((b"ix00" if s == 0 else b"ix01") + struct.pack("<IHBBI4sQI", 24 + 8 * len(chunks), 2, 0, 1, len(chunks),
                                                                      cid, base, 0))
            f.write(b"".join(struct.pack("<II", off - base, size) for off, size, _ in chunks))
            self._segments[s].append((at, 32 + 8 * len(chunks), sum(d for _, _, d in chunks)))
            if len(self._segments[s]) > _SUPER_ENTRIES:
                raise RuntimeError(f"more than {_SUPER_ENTRIES} RIFF segments; raise segment_bytes")
        self._patch_size(self._movi)
        if self._first:
            f.write(b"idx1" + struct.pack("<I", 16 * len(self._idx1)))
            f.write(b"".join(struct.pack("<4sIII", cid, _KEYFRAME, off - self._movi - 8, size)
                             for cid, off, size in self._idx1))
            self._first_frames = self.frames
        self._patch_size(self._riff)

    def _chunk(self, stream: int, data: bytes, duration: int):
        size = len(data)
        need = 8 + size + (size & 1) + 8 * 8 + 64            # the chunk and room for its index entries
        if self._first:
            need += 16 * (len(self._idx1) + 1)
        if self._f.tell() - self._riff + need > self.segment_bytes and any(self._chunks[:self._streams]):
            self._close_segment()
            self._open_segment(first=False)
        cid = b"00dc" if stream == 0 else b"01wb"
        at = self._f.tell()
        self._f.write(cid + struct.pack("<I", size) + data + (b"\0" if size & 1 else b""))
        self._chunks[stream].append((at + 8, size, duration))
        if self._first:
            self._idx1.append((cid, at, size))
        self._max_chunk = max(self._max_chunk, size)

    # -- public -----------------------------------------------------------------------------------------------------
    def write_frame(self, jpeg: bytes) -> None:
        self._chunk(0, bytes(jpeg), 1)
        self.frames += 1
        if self.audio_rate is not None:
            self._flush_audio(self._audio_end(self.frames))

    def _audio_end(self, frames: int) -> int:
        """floor(frames * audio_rate / fps), exactly."""
        scale, rate = self._rate()
        return frames * self.audio_rate * scale // rate

    def write_audio(self, samples) -> None:
        if self.audio_rate is None:
            raise RuntimeError("this writer has no audio stream (audio_rate=None)")
        a = np.asarray(samples)
        if a.dtype != self.dtype:
            raise ValueError(f"audio samples must be {np.dtype(self.dtype).name} (got {a.dtype})")
        a = a.reshape(-1, self.channels)
        if len(a):
            self._pending.append(np.ascontiguousarray(a))
            self._pending_n += len(a)

    def _flush_audio(self, upto: int) -> None:
        """Writes buffered audio up to sample frame ``upto`` as one chunk."""
        take = min(upto - self.samples, self._pending_n)
        if take <= 0:
            return
        buf = np.concatenate(self._pending) if len(self._pending) > 1 else self._pending[0]
        self._chunk(1, buf[:take].tobytes(), take)
        rest = buf[take:]
        self._pending = [rest] if len(rest) else []
        self._pending_n = len(rest)
        self.samples += take

    def close(self) -> None:
        if self._f.closed:
            return
        if self.audio_rate is not None:
            self._flush_audio(self._audio_end(self.frames))
        self._close_segment()
        f = self._f
        end = f.tell()
        scale, rate = self._rate()
        first = getattr(self, "_first_frames", self.frames)
        f.seek(self._avih)
        f.write(struct.pack("<IIIIIIIIII", int(round(1e6 * scale / rate)), 0, 0, 0x10 | 0x100, first, 0, self._streams,
                            self._max_chunk + 8, self.width, self.height))
        for s in range(self._streams):
            f.seek(self._strh[s])
            if s == 0:
                f.write(struct.pack("<4s4sIHHIIIIIIiIhhhh", b"vids", b"MJPG", 0, 0, 0, 0, scale, rate, 0, self.frames,
                                    self._max_chunk, -1, 0, 0, 0, self.width, self.height))
            else:
                f.write(struct.pack("<4s4sIHHIIIIIIiIhhhh", b"auds", b"\0\0\0\0", 0, 0, 0, 0, self.block_align,
                                    self.audio_rate * self.block_align, 0, self.samples, self._max_chunk, -1,
                                    self.block_align, 0, 0, 0, 0))
            segs = self._segments[s]
            f.seek(self._indx[s] + 8)
            f.write(struct.pack("<HBBI4sIII", 4, 0, 0, len(segs), b"00dc" if s == 0 else b"01wb", 0, 0, 0))
            f.write(b"".join(struct.pack("<QII", off, size, dur) for off, size, dur in segs))
        f.seek(self._dmlh)
        f.write(struct.pack("<I", self.frames))
        f.seek(end)
        f.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


# ---- GPU-encoded frames into the file: whole clips and live streams ------------------------------------------------

class _JpegSink:
    """A writer thread fed with encoded batches: for each item it waits (polling, so the host never blocks in a CUDA
    synchronisation) for the event recorded after the encoding and the copy of ``sizes`` to pinned memory, copies exactly
    ``sizes[i]`` bytes of each file to the host on a stream of its own, and hands the files (and the audio of the item) to
    ``MjpegAviWriter`` and to ``frames_dir`` as ``<prefix><j+1>.jpg``."""

    def __init__(self, writer: Optional[MjpegAviWriter], device: torch.device, frames_dir: Optional[str] = None,
                 prefix: str = "pred_"):
        self.writer, self.frames_dir, self.prefix = writer, frames_dir, prefix
        self.device = device
        self.copy_stream = torch.cuda.Stream(device)
        self.q: "queue.Queue" = queue.Queue()
        self.error: Optional[BaseException] = None
        self.busy_seconds = 0.0
        self.frames = 0
        self.thread = threading.Thread(target=self._run, daemon=True)
        self.thread.start()

    @staticmethod
    def _wait(ev: torch.cuda.Event) -> None:
        while not ev.query():
            time.sleep(5e-5)

    def _run(self):
        try:
            while True:
                item = self.q.get()
                if item is None:
                    return
                ev, data, sizes_host, n, audio, release = item
                self._wait(ev)
                t0 = time.perf_counter()
                sizes = sizes_host[:n].tolist()
                host = torch.empty(max(sum(sizes), 1), dtype=torch.uint8, pin_memory=True)
                with torch.cuda.stream(self.copy_stream):
                    self.copy_stream.wait_event(ev)
                    at = 0
                    for i, sz in enumerate(sizes):
                        host[at:at + sz].copy_(data[i, :sz], non_blocking=True)
                        at += sz
                    done = torch.cuda.Event()
                    done.record(self.copy_stream)
                self._wait(done)
                if release is not None:
                    release.set()
                if audio is not None and self.writer is not None:
                    self.writer.write_audio(audio)    # buffered; each frame below flushes the audio of its interval
                buf, at = host.numpy(), 0
                for sz in sizes:
                    jpg = buf[at:at + sz].tobytes()
                    at += sz
                    if self.frames_dir is not None:
                        with open(os.path.join(self.frames_dir, f"{self.prefix}{self.frames + 1}.jpg"), "wb") as f:
                            f.write(jpg)
                    if self.writer is not None:
                        self.writer.write_frame(jpg)
                    self.frames += 1
                self.busy_seconds += time.perf_counter() - t0
        except BaseException as exc:      # noqa: BLE001 - surfaced by close()
            self.error = exc

    def put(self, ev, data, sizes_host, n, audio=None, release=None) -> None:
        if self.error is not None:
            raise self.error
        self.q.put((ev, data, sizes_host, n, audio, release))

    def close(self) -> None:
        self.q.put(None)
        self.thread.join()
        if self.writer is not None:
            self.writer.close()
        if self.error is not None:
            raise self.error


def _encode_and_queue(enc, images, slot, sink, audio=None):
    """Encodes ``images`` into the slot's device buffers on the current stream, copies ``sizes`` into the slot's pinned
    buffer behind it, records an event and queues the batch for ``sink``."""
    n = images.shape[0]
    h, w = int(images.shape[1]), int(images.shape[2])
    c = 3 if images.dim() == 4 else 1
    dev = images.device
    stride = enc.max_bytes(h, w, c)
    if slot.get("data") is None or slot["data"].shape[0] < n or slot["data"].shape[1] != stride:
        slot["data"] = torch.empty((max(n, 1), stride), dtype=torch.uint8, device=dev)
        slot["sizes"] = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        slot["sizes_host"] = torch.empty(max(n, 1), dtype=torch.int32, pin_memory=True)
    slot["ws"] = _lib.reserve(slot.get("ws"), enc.workspace_bytes(n, h, w, c), dev)
    if n:
        batch = enc.encode_into(images, slot["data"], slot["sizes"], slot["ws"])
        slot["sizes_host"][:n].copy_(batch.sizes, non_blocking=True)
    ev = torch.cuda.Event()
    ev.record(torch.cuda.current_stream(dev))
    sink.put(ev, slot["data"], slot["sizes_host"], n, audio, slot.get("free"))


def render_to_mjpeg(net, landmarks, shoulders, cand, output_path: str, size: tuple = (512, 512), fps: float = 60,
                    batch: int = 32, quality: int = 75, audio=None, audio_rate: int = 16000,
                    feature_maps_path: Optional[str] = None, frames_dir: Optional[str] = None,
                    precision: Optional[str] = None) -> dict:
    """Render a clip from its landmark tracks into a Motion-JPEG AVI with its audio, encoding on the GPU.

    Arguments as ``render_to_video``; ``audio``: the clip's samples (numpy float32 ``[n]`` or ``[n, channels]``, or
    int16), written at ``audio_rate`` and cut to the video's length like demo.py's ``ffmpeg -shortest``.  Each batch is
    rasterised and rendered to uint8 frames on a compute stream, encoded there by ``JpegEncoder`` (PIL's bytes at
    ``quality``), and only ``sizes[i]`` bytes per frame cross PCIe; a writer thread builds the file.
    ``feature_maps_path``: the rasterised maps as a second MJPEG AVI of one-component JPEGs of ``np.uint8(map * 255)``.
    ``frames_dir``: also write ``pred_<j+1>.jpg`` (and ``input_<j+1>.jpg`` for the maps) with demo.py's bytes.
    Returns ``{"frames", "seconds", "encode_seconds", "writer", "bytes"}``."""
    from .jpeg import JpegEncoder
    n = int(landmarks.shape[0])
    w, h = int(size[0]), int(size[1])
    dev = cand.device
    lm = _tracks(landmarks, dev).to(dev, non_blocking=True)
    sh = None if shoulders is None else _tracks(shoulders, dev).to(dev, non_blocking=True)
    a = None if audio is None else np.asarray(audio)
    channels = 1 if a is None or a.ndim == 1 else int(a.shape[1])
    t0 = time.perf_counter()
    writer = MjpegAviWriter(output_path, (w, h), fps, None if a is None else audio_rate, channels,
                            "s16" if a is not None and a.dtype == np.int16 else "f32")
    if a is not None:
        writer.write_audio(a)                         # interleaved as the frames arrive, cut on close
    sink = _JpegSink(writer, dev, frames_dir, "pred_")
    fsink = None
    if feature_maps_path is not None or frames_dir is not None:
        fwriter = None if feature_maps_path is None else MjpegAviWriter(feature_maps_path, (w, h), fps)
        fsink = _JpegSink(fwriter, dev, frames_dir, "input_")
    enc = JpegEncoder(dev, quality)
    compute = torch.cuda.Stream(dev)
    compute.wait_stream(torch.cuda.current_stream(dev))
    slots = [{"free": threading.Event()} for _ in range(2)]
    fslots = [{"free": threading.Event()} for _ in range(2)]
    for s in slots + fslots:
        s["free"].set()
    fm = torch.empty((batch, 1, h, w), dtype=torch.float32, device=dev)
    frames = torch.empty((batch, h, w, 3), dtype=torch.uint8, device=dev)
    try:
        with torch.cuda.stream(compute):
            for bi, off in enumerate(range(0, n, batch)):
                ln = min(batch, n - off)
                slot, fslot = slots[bi & 1], fslots[bi & 1]
                slot["free"].wait()                   # the writer thread has copied this slot's files out
                slot["free"].clear()
                net.draw_feature_maps(lm[off:off + ln], None if sh is None else sh[off:off + ln], (w, h), out=fm[:ln])
                if fsink is not None:
                    fslot["free"].wait()
                    fslot["free"].clear()
                    _encode_and_queue(enc, (fm[:ln, 0] * 255.0).to(torch.uint8), fslot, fsink)
                cd = cand[off:off + ln] if cand.shape[0] == n and n > 1 else cand[:1]
                net.render(fm[:ln], cd, out=frames[:ln], precision=precision, _uint8=True)
                _encode_and_queue(enc, frames[:ln], slot, sink)
    finally:
        sink.close()
        if fsink is not None:
            fsink.close()
    torch.cuda.current_stream(dev).wait_stream(compute)
    return {"frames": n, "seconds": time.perf_counter() - t0, "encode_seconds": sink.busy_seconds,
            "writer": f"MJPG q{quality} {fps:g} fps {w}x{h}", "bytes": os.path.getsize(output_path)}


class PortraitRecorder:
    """Records a ``PortraitStream`` into a Motion-JPEG AVI with its audio while it plays.

    ``push(samples)`` forwards to ``portrait_stream.push`` and returns its ``PortraitFrames`` unchanged; the frames are
    encoded on the same CUDA stream (``JpegEncoder``, PIL's bytes at ``quality``), and a writer thread waits for them,
    copies exactly their bytes and writes them with the pushed audio (at ``audio_rate`` / ``audio_channels`` as given: a
    stream that resamples records its native-rate input).  Pushes make no host synchronisation, and after the first push
    of a size the device memory stays the same; ``finish()`` finishes the stream, flushes and closes the file and
    returns the last ``PortraitFrames``."""

    _RING = 4                                          # pushes the writer thread may lag behind before push waits for it

    def __init__(self, portrait_stream, path: str, quality: int = 75, fps: float = 60, audio_rate: int = 16000,
                 audio_channels: int = 1, audio_format: str = "f32"):
        from .jpeg import JpegEncoder
        self.stream = portrait_stream
        self._enc = JpegEncoder(portrait_stream._cand.device, quality)
        self._dev = self._enc.device
        self._path, self._fps = path, fps
        self._audio = (audio_rate, audio_channels, audio_format)
        self._dtype = np.float32 if audio_format == "f32" else np.int16
        self._sink = None
        self._slots = [{"free": threading.Event()} for _ in range(self._RING)]
        for s in self._slots:
            s["free"].set()
        self._pushes = 0

    def _audio_copy(self, samples):
        if isinstance(samples, torch.Tensor) and samples.is_cuda:
            host = torch.empty(samples.shape, dtype=samples.dtype, pin_memory=True)
            host.copy_(samples, non_blocking=True)    # lands before the event recorded after the encoding
            return host.numpy()
        return np.array(torch.as_tensor(samples).numpy() if isinstance(samples, torch.Tensor) else samples,
                        dtype=self._dtype, copy=True)

    def _record(self, out, samples) -> None:
        if self._sink is None:
            w, h = self.stream._size
            self._sink = _JpegSink(MjpegAviWriter(self._path, (w, h), self._fps, *self._audio), self._dev)
        slot = self._slots[self._pushes % self._RING]
        self._pushes += 1
        slot["free"].wait()
        slot["free"].clear()
        audio = None if samples is None else self._audio_copy(samples)
        if audio is not None and audio.dtype != self._dtype:
            audio = audio.astype(self._dtype)
        _encode_and_queue(self._enc, out.frames, slot, self._sink, audio)

    def push(self, samples):
        out = self.stream.push(samples)
        self._record(out, samples)
        return out

    def finish(self):
        out = self.stream.finish()
        self._record(out, None)
        self._sink.close()
        return out
