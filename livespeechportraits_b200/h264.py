"""Frames -> H.264 on the GPU (include/lspv.h): Constrained Baseline access units in Annex B, each decoding in any
conforming decoder to exactly the reconstruction the encoder keeps.  The H100 has no NVENC; this runs on the SMs.

``H264Encoder.encode(images)`` codes a whole clip; ``H264Encoder.stream()`` codes a live session push by push, and the
pushes' access units concatenate to the whole clip's.  The raw elementary stream (``.h264``, what an RTP / MPEG-TS
packetiser or ``ffplay -f h264`` takes) is ``b"".join(batch.to_bytes())``."""
from __future__ import annotations

import ctypes as C
import dataclasses
from typing import List

import torch

from . import _lib


@dataclasses.dataclass
class H264Batch:
    """``n`` access units on the device: unit ``i`` is ``data[i, :sizes[i]]``, an IDR when ``is_idr[i]``."""
    data: torch.Tensor            # [n, stride] uint8, stride >= H264Encoder.max_bytes
    sizes: torch.Tensor           # [n] int32
    is_idr: torch.Tensor          # [n] uint8

    def to_bytes(self) -> List[bytes]:
        """The access units on the host (synchronises with the encoding)."""
        sizes = self.sizes.cpu().tolist()
        if not sizes:
            return []
        data = self.data[:, :max(sizes)].cpu().numpy()
        return [bytes(data[i, :s]) for i, s in enumerate(sizes)]


class H264Encoder(_lib.Handle):
    """H.264 encoding of uint8 frames on the device, asynchronous on the current CUDA stream.

    ``qp`` is the fixed quantiser (0..51), ``gop`` the IDR period in frames, ``search`` the full-pel motion range and
    ``fps`` the frame rate written into the stream's timing (and used for its level).  Frames are ``[n, H, W, 3]`` RGB
    or ``[n, H, W]`` grey uint8 CUDA tensors, H and W multiples of 16."""
    prefix = "lspv"
    what = "the H.264 encoder"

    def __init__(self, device=None, qp: int = 26, gop: int = 60, search: int = 16, fps: int = 60):
        super().__init__(device)
        self.qp, self.gop, self.search, self.fps = int(qp), int(gop), int(search), int(fps)
        self._create(self.qp, self.gop, self.search, self.fps)
        self._ws = None

    def _size(self, name: str, height: int, width: int) -> int:
        out = C.c_size_t()
        self.call(name, int(height), int(width), C.byref(out))
        return out.value

    def max_bytes(self, height: int, width: int) -> int:
        """``lspv_max_bytes``: no access unit of a ``height`` x ``width`` frame is longer."""
        return self._size("max_bytes", height, width)

    def state_bytes(self, height: int, width: int) -> int:
        return self._size("state_bytes", height, width)

    def workspace_bytes(self, height: int, width: int) -> int:
        return self._size("workspace_bytes", height, width)

    def new_state(self, height: int, width: int) -> torch.Tensor:
        """A fresh encoder state (the first call on it must start at a frame index that is a multiple of ``gop``)."""
        return torch.zeros(self.state_bytes(height, width), dtype=torch.uint8, device=self.device)

    @staticmethod
    def _shape(images: torch.Tensor):
        if images.dtype != torch.uint8 or not images.is_cuda or images.dim() not in (3, 4) or \
                (images.dim() == 4 and images.shape[3] != 3):
            raise ValueError("images must be a uint8 CUDA tensor [n, H, W, 3] (RGB) or [n, H, W] (grey)")
        n, h, w = images.shape[:3]
        return int(n), int(h), int(w), 3 if images.dim() == 4 else 1

    def encode(self, images: torch.Tensor) -> H264Batch:
        """A whole clip: frames 0 .. n-1 from a fresh state."""
        _, h, w, _ = self._shape(images)
        return self.encode_at(images, 0, self.new_state(h, w))

    def encode_at(self, images: torch.Tensor, f0: int, state: torch.Tensor) -> H264Batch:
        """Frames ``f0 .. f0 + n - 1`` from ``state`` (what the call that ended at ``f0`` left); updates ``state``."""
        n, h, w, _ = self._shape(images)
        data = torch.empty((n, self.max_bytes(h, w)), dtype=torch.uint8, device=self.device)
        sizes = torch.empty(n, dtype=torch.int32, device=self.device)
        idr = torch.empty(n, dtype=torch.uint8, device=self.device)
        return self.encode_into(images, f0, state, data, sizes, idr)

    def encode_into(self, images: torch.Tensor, f0: int, state: torch.Tensor, out: torch.Tensor, sizes: torch.Tensor,
                    is_idr: torch.Tensor) -> H264Batch:
        """``encode_at`` into caller-owned ``out`` ([>= n, stride >= max_bytes] uint8, rows contiguous), ``sizes``
        ([>= n] int32) and ``is_idr`` ([>= n] uint8).  Returns the views of the first n rows."""
        n, h, w, c = self._shape(images)
        images = images.contiguous()
        if state.dtype != torch.uint8 or state.numel() < self.state_bytes(h, w):
            raise ValueError("state must be a uint8 tensor of state_bytes(H, W) bytes")
        if out.dtype != torch.uint8 or out.dim() != 2 or out.shape[0] < n or out.stride(1) != 1 or \
                sizes.dtype != torch.int32 or not sizes.is_contiguous() or sizes.shape[0] < n or \
                is_idr.dtype != torch.uint8 or not is_idr.is_contiguous() or is_idr.shape[0] < n:
            raise ValueError("out must be uint8 [>= n, stride] with contiguous rows, sizes int32 [>= n], is_idr uint8 [>= n]")
        for t in (images, state, out, sizes, is_idr):
            if t.device != self.device:
                raise ValueError(f"every buffer must be on {self.device}")
        self._ws = _lib.reserve(self._ws, self.workspace_bytes(h, w), self.device)
        with self.cuda_stream() as s:
            self.call("encode", images.data_ptr(), n, h, w, c, int(f0), state.data_ptr(), out.data_ptr(), out.stride(0),
                      sizes.data_ptr(), is_idr.data_ptr(), self._ws.data_ptr(), self._ws.numel(), s)
        return H264Batch(out[:n], sizes[:n], is_idr[:n])

    def stream(self) -> "H264Stream":
        return H264Stream(self)


class H264Stream:
    """A live session: ``push(images)`` returns the access units of the frames pushed, at once (there are no B frames,
    so nothing waits for later frames); ``finish()`` returns an empty batch.  The concatenation equals
    ``encoder.encode`` of all frames."""

    def __init__(self, encoder: H264Encoder):
        self.encoder = encoder
        self.frames = 0
        self.state = None
        self._shape = None

    def _begin(self, images: torch.Tensor) -> int:
        n, h, w, _ = self.encoder._shape(images)
        if self._shape is None:
            self._shape = (h, w)
            self.state = self.encoder.new_state(h, w)
        elif self._shape != (h, w):
            raise ValueError(f"frames of one stream keep their size {self._shape} (got {(h, w)})")
        return n

    def push(self, images: torch.Tensor) -> H264Batch:
        n = self._begin(images)
        out = self.encoder.encode_at(images, self.frames, self.state)
        self.frames += n
        return out

    def push_into(self, images: torch.Tensor, out: torch.Tensor, sizes: torch.Tensor, is_idr: torch.Tensor) -> H264Batch:
        """``push`` into caller-owned buffers (as ``H264Encoder.encode_into``)."""
        n = self._begin(images)
        batch = self.encoder.encode_into(images, self.frames, self.state, out, sizes, is_idr)
        self.frames += n
        return batch

    def finish(self) -> H264Batch:
        dev = self.encoder.device
        return H264Batch(torch.empty((0, 1), dtype=torch.uint8, device=dev), torch.empty(0, dtype=torch.int32, device=dev),
                         torch.empty(0, dtype=torch.uint8, device=dev))
