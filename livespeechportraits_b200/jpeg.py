"""Frames -> .jpg files on the GPU (include/lspj.h): each file equals, byte for byte, what PIL's ``Image.save(f, "JPEG",
quality=q)`` writes for the same uint8 image - demo.py's ``visualizer.save_images`` at its defaults is quality 75."""
from __future__ import annotations

import ctypes as C
import dataclasses
from typing import List

import torch

from . import _lib


@dataclasses.dataclass
class JpegBatch:
    """``n`` files on the device: file ``i`` is ``data[i, :sizes[i]]``."""
    data: torch.Tensor            # [n, stride] uint8, stride >= JpegEncoder.max_bytes
    sizes: torch.Tensor           # [n] int32

    def to_bytes(self) -> List[bytes]:
        """The files on the host (synchronises with the encoding)."""
        sizes = self.sizes.cpu().tolist()
        return [bytes(self.data[i, :s].cpu().numpy()) for i, s in enumerate(sizes)]


class JpegEncoder(_lib.Handle):
    """Baseline JPEG encoding of uint8 frames on the device, asynchronous on the current CUDA stream.

    ``encode(images)`` takes ``[n, H, W, 3]`` RGB (tensor2im's layout) or ``[n, H, W]`` grey, H and W multiples of 16,
    and allocates its outputs and a workspace of its own, so calls on one encoder may run on several CUDA streams at
    once.  ``encode_into`` writes into caller-owned buffers with a caller-owned workspace, which calls that may overlap
    must not share."""
    prefix = "lspj"
    what = "the JPEG encoder"

    def __init__(self, device=None, quality: int = 75):
        super().__init__(device)
        if not 1 <= int(quality) <= 100:
            raise ValueError(f"quality must be in [1, 100] (got {quality})")
        self.quality = int(quality)
        self._create()

    def max_bytes(self, height: int, width: int, components: int = 3) -> int:
        """``lspj_max_bytes``: no file of a ``height`` x ``width`` frame is longer."""
        out = C.c_size_t()
        self.call("max_bytes", int(height), int(width), int(components), C.byref(out))
        return out.value

    def encode(self, images: torch.Tensor) -> JpegBatch:
        n, h, w, c = _lib.frame_shape(images)
        data = torch.empty((n, self.max_bytes(h, w, c)), dtype=torch.uint8, device=self.device)
        sizes = torch.empty(n, dtype=torch.int32, device=self.device)
        return self.encode_into(images, data, sizes, self.workspace(n, h, w, c))

    def encode_into(self, images: torch.Tensor, out: torch.Tensor, sizes: torch.Tensor, ws: torch.Tensor) -> JpegBatch:
        """Encodes into ``out`` ([>= n, stride] uint8, rows contiguous), ``sizes`` ([>= n] int32) with the workspace ``ws``
        (uint8, at least ``workspace_bytes(n, H, W, components)`` bytes).  Returns the views of the first n rows."""
        n, h, w, c = _lib.frame_shape(images)
        images = images.contiguous()
        if out.dtype != torch.uint8 or out.dim() != 2 or out.shape[0] < n or out.stride(1) != 1 or \
                sizes.dtype != torch.int32 or not sizes.is_contiguous() or sizes.shape[0] < n or ws.dtype != torch.uint8:
            raise ValueError("out must be uint8 [>= n, stride] with contiguous rows, sizes int32 [>= n], ws uint8")
        for t in (images, out, sizes, ws):
            if t.device != self.device:
                raise ValueError(f"every buffer must be on {self.device}")
        with self.cuda_stream() as s:
            self.call("encode", images.data_ptr(), n, h, w, c, self.quality, out.data_ptr(), out.stride(0),
                      sizes.data_ptr(), ws.data_ptr(), ws.numel(), s)
        return JpegBatch(out[:n], sizes[:n])
