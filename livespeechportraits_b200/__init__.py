"""H100-native implementation of LiveSpeechPortraits' per-frame renderer (``Feature2Face_G``) and the steps either
side of it.  Public names:

* ``Feature2Face_G`` / ``install`` - drop-in for ``models/feature2face_G.py`` (generator.py)
* ``ClipRenderer`` - batched host-to-host render loop (pipeline.py)
* ``ShardedRenderer`` / ``partition`` - one process per GPU, frames partitioned, one gather (parallel.py)
* ``render_to_video`` - landmark tracks -> video file, the demo.py loop body without JPEGs (video.py)
* ``JpegEncoder`` - uint8 frames -> PIL's .jpg bytes on the GPU (jpeg.py); ``render_to_mjpeg`` / ``PortraitRecorder`` /
  ``MjpegAviWriter`` - whole clips and live streams into Motion-JPEG AVI files with their audio (video.py)
* ``ManifoldProjector`` / ``install_manifold`` - APC feature KNN + LLE projection, drop-in for funcs/utils.py (manifold.py)

Importing the package does not touch CUDA; the native library is loaded (and built if missing) on first use.
"""
from .generator import Feature2Face_G, install  # noqa: F401
from .manifold import ManifoldProjector  # noqa: F401
from .manifold import install as install_manifold  # noqa: F401
from .parallel import ShardedRenderer, partition  # noqa: F401
from .pipeline import ClipRenderer  # noqa: F401
from .jpeg import JpegBatch, JpegEncoder  # noqa: F401
from .video import MjpegAviWriter, PortraitRecorder, render_to_mjpeg, render_to_video  # noqa: F401

__all__ = ["Feature2Face_G", "install", "ClipRenderer", "ShardedRenderer", "partition", "render_to_video", "ManifoldProjector",
           "install_manifold", "JpegEncoder", "JpegBatch", "render_to_mjpeg", "PortraitRecorder", "MjpegAviWriter"]
