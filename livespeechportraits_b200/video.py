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
import subprocess
import threading
import time
from typing import Optional

import numpy as np
import torch

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
