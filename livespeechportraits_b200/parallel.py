"""Frame-sharded rendering across GPUs: one process per GPU, weights replicated, frames partitioned.

The reference's only multi-GPU hook is ``nn.DataParallel`` (models/networks.py:392-401), single process, with a
gather of the outputs on device 0.  Frames are independent (eval-mode BatchNorm, no temporal state:
demo.py:260-266), so the layout is: contiguous block partition of the clip's frames over the ranks, no
data-path collective while rendering, and ONE exchange step - every rank ends up with every frame (the
all-gather BASELINE.json names).

Two implementations of the exchange, chosen by ``gather=``:

``"ce"``  (default where it works) - the clip buffer ``[n_total, ...]`` is allocated as *symmetric memory*
    (``torch.distributed._symmetric_memory``: the same allocation mapped into every rank over NVLink).  The tail
    kernel of each chunk writes this rank's frames straight into its own block of the buffer; the chunk is then
    PUSHED into the same block of every peer's buffer with peer-to-peer ``cudaMemcpyAsync`` on side streams - the
    copy engines move the bytes, no SM and no NCCL kernel runs next to the persistent conv kernels (round-1
    finding: the SM-resident NCCL all-gather slowed the convs by 9 % at 8 GPUs).  One cross-rank barrier at the end
    of the clip (or per chunk when frames are delivered to the host as they complete).
``"mc"``  (opt-in, fp32 frames) - same symmetric clip buffer, but the tail kernel's output address is the buffer's NVLink
    *multicast* mapping (NVLS): every float2 store of the conv epilogue lands in all ranks' buffers through the switch.  No
    copy of any kind follows the conv kernel - the collective is fused into it.  Needs ``render_ptr_fn`` (a function that
    renders to a raw device address, ``Feature2Face_G.render_into_ptr``) and multicast support on the node.
``"nccl"`` - ``all_gather_into_tensor`` per chunk on a side stream into a double-buffered staging tensor and a copy
    into clip order (the round-1 path; also what runs on CPU/gloo in the tests).

Frames are fp32 ``[3,H,W]`` (the reference's ``fake_pred``) or, with ``uint8=True``, uint8 ``[H,W,3]`` images
(``util.tensor2im`` fused into the tail kernel - a quarter of the bytes).
"""
from __future__ import annotations

import contextlib
from typing import Callable, Dict, List, Optional, Tuple

import torch
import torch.distributed as dist


def partition(n_items: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous balanced block partition: the first ``n_items % world`` ranks get one extra item."""
    if world < 1 or not (0 <= rank < world) or n_items < 0:
        raise ValueError("bad partition arguments")
    base, extra = divmod(n_items, world)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


def chunk_schedule(n_local_max: int, chunk: int) -> List[Tuple[int, int]]:
    """[(offset, length)] over the LONGEST shard; shorter shards render fewer frames in the last chunk(s)."""
    if chunk < 1:
        raise ValueError("chunk must be >= 1")
    return [(o, min(chunk, n_local_max - o)) for o in range(0, n_local_max, chunk)]


class ShardedRenderer:
    """Renders this rank's shard chunk by chunk and delivers the frames of every rank to every rank.

    ``render_fn(feature_maps[n,1,H,W], out[n,...]) -> None`` renders into ``out`` in place (on GPU this is
    ``Feature2Face_G.render(fm, cand, out=out)`` / ``render_image``; tests on CPU/gloo pass a torch function).
    """

    def __init__(self, render_fn: Callable[[torch.Tensor, torch.Tensor], None], group=None, chunk: int = 32,
                 uint8: bool = False, gather: str = "auto", copy_streams: int = 4,
                 render_ptr_fn: Optional[Callable[[torch.Tensor, int], None]] = None):
        if gather not in ("auto", "ce", "mc", "nccl"):
            raise ValueError("gather must be 'auto', 'ce', 'mc' or 'nccl'")
        if gather == "mc" and (render_ptr_fn is None or uint8):
            raise ValueError("gather='mc' needs render_ptr_fn and fp32 frames (multicast stores are 8-byte float2 stores)")
        self.render_ptr_fn = render_ptr_fn
        self.render_fn = render_fn
        self.group = group
        self.chunk = int(chunk)
        self.uint8 = bool(uint8)
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.gather_request = gather
        self.gather_mode: Optional[str] = None        # decided at the first gathered render ("ce" or "nccl")
        self.gather_fallback_reason: Optional[str] = None
        self._n_copy_streams = max(1, int(copy_streams))
        self._symm: Dict[tuple, tuple] = {}           # (n_total, h, w, uint8) -> (clip tensor, handle, peer views)
        self._streams: Optional[List[torch.cuda.Stream]] = None

    # ------------------------------------------------------------------ shapes
    def _frame_shape(self, h: int, w: int) -> Tuple[int, ...]:
        return (h, w, 3) if self.uint8 else (3, h, w)

    def _dtype(self) -> torch.dtype:
        return torch.uint8 if self.uint8 else torch.float32

    # ------------------------------------------------------------------ symmetric clip buffer (copy-engine mode)
    def _symmetric_clip(self, n_total: int, h: int, w: int, dev: torch.device):
        """Clip buffer mapped into every rank + views of every peer's copy.  Collective: every rank calls it with the same
        arguments in the same order.  Raises if symmetric memory is unavailable (caller falls back to NCCL)."""
        key = (h, w, self.uint8)
        hit = self._symm.get(key)
        if hit is not None and hit[0] >= n_total:     # one allocation serves every clip up to its capacity
            cap, clip, hdl, peers = hit
            return clip[:n_total], hdl, [p_[:n_total] for p_ in peers]
        import torch.distributed._symmetric_memory as symm_mem
        if self._symm:
            torch.cuda.synchronize(dev)               # nothing in flight may still touch a buffer that is about to be released
        self._symm.pop(key, None)                     # growing: release the smaller buffer first
        shape = (n_total,) + self._frame_shape(h, w)
        clip = symm_mem.empty(*shape, dtype=self._dtype(), device=dev)
        grp = self.group if self.group is not None else dist.group.WORLD
        hdl = symm_mem.rendezvous(clip, grp)
        peers = [clip if r == self.rank else hdl.get_buffer(r, shape, self._dtype()) for r in range(self.world)]
        if len(self._symm) >= 2:                      # a clip buffer is large: keep at most two frame shapes alive
            self._symm.pop(next(iter(self._symm)))
        self._symm[key] = (n_total, clip, hdl, peers)
        return clip, hdl, peers

    def prepare(self, n_total: int, height: int, width: int, device: torch.device) -> str:
        """Collective, optional: decide the exchange mode and allocate + rendezvous the symmetric clip buffer for clips of up
        to ``n_total`` frames now (hundreds of milliseconds for a multi-GB buffer) instead of inside the first ``render``.
        Returns the mode that will run ("ce", "mc" or "nccl")."""
        if self.world == 1:
            return "local"
        dev = torch.device(device)
        mode = self._decide_mode(n_total, height, width, dev)
        if mode in ("ce", "mc"):
            self._symmetric_clip(n_total, height, width, dev)       # grows the buffer if an earlier clip was shorter
        return mode

    def _decide_mode(self, n_total: int, h: int, w: int, dev: torch.device) -> str:
        """"ce" needs CUDA + symmetric memory on every rank; agreement is reached with one tiny all-reduce."""
        if self.gather_mode is not None:
            return self.gather_mode
        mode, why = "nccl", None
        if self.gather_request in ("auto", "ce", "mc") and dev.type == "cuda" and self.world > 1:
            ok = 1
            try:
                _, hdl_, _ = self._symmetric_clip(n_total, h, w, dev)
                if self.gather_request == "mc" and not (hdl_.has_multicast_support and int(hdl_.multicast_ptr) != 0):
                    raise RuntimeError("the symmetric allocation has no NVLink multicast mapping on this node")
            except Exception as exc:          # noqa: BLE001 - any failure means "not available here"
                ok, why = 0, f"{type(exc).__name__}: {exc}"
            flag = torch.tensor([ok], device=dev, dtype=torch.int32)
            dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.group)
            if int(flag.item()) == 1:
                mode = "mc" if self.gather_request == "mc" else "ce"
            else:
                why = why or "symmetric memory unavailable on another rank"
                self._symm.clear()
                if self.gather_request in ("ce", "mc"):
                    raise RuntimeError(f"gather={self.gather_request!r} requested but it is unavailable here: {why}")
        elif self.gather_request in ("ce", "mc"):
            raise RuntimeError(f"gather={self.gather_request!r} needs CUDA devices and world_size > 1")
        self.gather_mode, self.gather_fallback_reason = mode, why
        return mode

    def _copy_streams(self, dev: torch.device) -> List[torch.cuda.Stream]:
        if self._streams is None:
            self._streams = [torch.cuda.Stream(device=dev) for _ in range(self._n_copy_streams)]
        return self._streams

    # ------------------------------------------------------------------ render
    def render(self, n_total: int, local_feature_maps: torch.Tensor, gather: bool = True,
               host_out: Optional[torch.Tensor] = None, to_host: bool = False) -> torch.Tensor:
        """``local_feature_maps``: this rank's block ``partition(n_total, world, rank)`` of the clip, on this rank's device.

        Returns ``[n_total, ...]`` (every rank holds all frames, frame order = clip order) when ``gather``, else this
        rank's ``[n_local, ...]``.  ``to_host=True`` (a COLLECTIVE choice: pass the same value on every rank) delivers the
        gathered frames to rank 0's ``host_out`` (pinned ``[n_total, ...]``, needed on rank 0 only) chunk by chunk while
        later chunks render; the call returns after the last copy has landed.  In "ce" mode the returned tensor is the
        renderer's symmetric clip buffer: it is overwritten by the next ``render`` of the same shape.
        """
        if host_out is not None and not to_host and self.world > 1:
            raise ValueError("host_out needs to_host=True on EVERY rank (the per-chunk completion barrier is collective)")
        if to_host and self.rank == 0 and host_out is None and gather:
            raise ValueError("to_host=True: rank 0 must supply host_out")
        if self.rank != 0:
            host_out = None
        start, stop = partition(n_total, self.world, self.rank)
        n_local = stop - start
        if local_feature_maps.shape[0] != n_local:
            raise ValueError(f"rank {self.rank} expected {n_local} frames, got {local_feature_maps.shape[0]}")
        dev = local_feature_maps.device
        h, w = local_feature_maps.shape[-2:]
        fshape, dt = self._frame_shape(h, w), self._dtype()
        if host_out is not None and (tuple(host_out.shape) != (n_total,) + fshape or host_out.dtype != dt):
            raise ValueError(f"host_out must be {dt} of shape {(n_total,) + fshape}")
        if not gather or self.world == 1:
            out = torch.empty((n_local,) + fshape, dtype=dt, device=dev)
            d2h = torch.cuda.Stream(device=dev) if (host_out is not None and dev.type == "cuda") else None
            for off, ln in chunk_schedule(n_local, self.chunk):
                self.render_fn(local_feature_maps[off:off + ln], out[off:off + ln])
                if host_out is not None and self.world == 1:
                    if d2h is not None:
                        d2h.wait_stream(torch.cuda.current_stream(dev))
                        with torch.cuda.stream(d2h):
                            host_out[off:off + ln].copy_(out[off:off + ln], non_blocking=True)
                    else:
                        host_out[off:off + ln].copy_(out[off:off + ln])
            if d2h is not None:
                d2h.synchronize()
            return out
        mode = self._decide_mode(n_total, h, w, dev)
        if mode in ("ce", "mc"):
            return self._render_ce(n_total, local_feature_maps, host_out, to_host, multicast=(mode == "mc"))
        return self._render_nccl(n_total, local_feature_maps, host_out)

    # ------------------------------------------------------------------ copy-engine push over symmetric memory
    def _render_ce(self, n_total: int, local_feature_maps: torch.Tensor, host_out: Optional[torch.Tensor],
                   to_host: bool, multicast: bool = False) -> torch.Tensor:
        dev = local_feature_maps.device
        h, w = local_feature_maps.shape[-2:]
        clip, hdl, peers = self._symmetric_clip(n_total, h, w, dev)
        start, stop = partition(n_total, self.world, self.rank)
        n_local = stop - start
        n_max = partition(n_total, self.world, 0)[1]
        bounds = [partition(n_total, self.world, r) for r in range(self.world)]
        cur = torch.cuda.current_stream(dev)
        streams = self._copy_streams(dev)
        others = [(self.rank + k) % self.world for k in range(1, self.world)]       # staggered: ranks start on different peers
        per_chunk_sync = bool(to_host)          # identical on every rank: the per-chunk barrier below is collective
        d2h = torch.cuda.Stream(device=dev) if (per_chunk_sync and self.rank == 0) else None
        # nobody may still be reading the previous clip out of this buffer / pushing into it
        hdl.barrier(channel=0)
        for off, ln in chunk_schedule(n_max, self.chunk):
            mine = max(0, min(ln, n_local - off))
            if mine > 0 and multicast:
                # the tail kernel stores through the multicast mapping: its float2 stores reach every rank's clip buffer
                frame_bytes = clip[0].numel() * clip.element_size()
                self.render_ptr_fn(local_feature_maps[off:off + mine], int(hdl.multicast_ptr) + (start + off) * frame_bytes)
            elif mine > 0:
                lo = start + off
                self.render_fn(local_feature_maps[off:off + mine], clip[lo:lo + mine])      # tail kernel -> clip buffer
                ready = torch.cuda.Event()
                ready.record(cur)
                for k, p in enumerate(others):
                    s = streams[k % len(streams)]
                    s.wait_event(ready)
                    with torch.cuda.stream(s):
                        peers[p][lo:lo + mine].copy_(clip[lo:lo + mine], non_blocking=True)  # P2P memcpy: copy engines
            if per_chunk_sync:
                # frames leave for the host as soon as every rank's share of the chunk has landed everywhere
                s0 = streams[0]
                for s in streams[1:]:
                    s0.wait_stream(s)
                s0.wait_stream(cur)
                with torch.cuda.stream(s0):
                    hdl.barrier(channel=1)
                    landed = torch.cuda.Event()
                    landed.record(s0)
                if d2h is not None:
                    d2h.wait_event(landed)
                    with torch.cuda.stream(d2h):
                        for (s_r, e_r) in bounds:
                            cnt = max(0, min(ln, (e_r - s_r) - off))
                            if cnt > 0:
                                host_out[s_r + off:s_r + off + cnt].copy_(clip[s_r + off:s_r + off + cnt], non_blocking=True)
        for s in streams:
            cur.wait_stream(s)
        hdl.barrier(channel=0)                        # every rank's pushes have landed everywhere
        if d2h is not None:
            d2h.synchronize()
        return clip

    # ------------------------------------------------------------------ NCCL / gloo all-gather
    def _render_nccl(self, n_total: int, local_feature_maps: torch.Tensor, host_out: Optional[torch.Tensor]) -> torch.Tensor:
        dev = local_feature_maps.device
        h, w = local_feature_maps.shape[-2:]
        fshape, dt = self._frame_shape(h, w), self._dtype()
        start, stop = partition(n_total, self.world, self.rank)
        n_local = stop - start
        n_max = partition(n_total, self.world, 0)[1]          # rank 0 holds the longest shard
        final = torch.empty((n_total,) + fshape, dtype=dt, device=dev)
        sched = chunk_schedule(n_max, self.chunk)
        bufs = [torch.empty((self.world, self.chunk) + fshape, dtype=dt, device=dev) for _ in range(2)]
        use_streams = dev.type == "cuda"
        comm = torch.cuda.Stream(device=dev) if use_streams else None
        d2h = torch.cuda.Stream(device=dev) if (use_streams and host_out is not None and self.rank == 0) else None
        if use_streams:                      # tensors allocated on the compute stream, also used on the comm stream
            final.record_stream(comm)
            for b_ in bufs:
                b_.record_stream(comm)
        done: List[Optional[torch.cuda.Event]] = [None, None]
        bounds = [partition(n_total, self.world, r) for r in range(self.world)]
        for ci, (off, ln) in enumerate(sched):
            buf = bufs[ci & 1]
            if use_streams and done[ci & 1] is not None:
                torch.cuda.current_stream(dev).wait_event(done[ci & 1])   # buffer free again
            mine = max(0, min(ln, n_local - off))
            if mine > 0:
                self.render_fn(local_feature_maps[off:off + mine], buf[self.rank, :mine])
            if use_streams:
                ready = torch.cuda.Event()
                ready.record(torch.cuda.current_stream(dev))
                comm.wait_event(ready)
                ctx = torch.cuda.stream(comm)
            else:
                ctx = contextlib.nullcontext()
            with ctx:
                flat = buf.view((self.world * self.chunk,) + fshape)
                dist.all_gather_into_tensor(flat, buf[self.rank], group=self.group)   # in place: slot = rank
                for r, (s, e) in enumerate(bounds):
                    cnt = max(0, min(ln, (e - s) - off))
                    if cnt > 0:
                        final[s + off:s + off + cnt].copy_(buf[r, :cnt], non_blocking=True)
                if use_streams:
                    ev = torch.cuda.Event()
                    ev.record(comm)
                    done[ci & 1] = ev
            if host_out is not None and self.rank == 0:
                if d2h is not None:
                    d2h.wait_event(done[ci & 1])
                    with torch.cuda.stream(d2h):
                        for (s, e) in bounds:
                            cnt = max(0, min(ln, (e - s) - off))
                            if cnt > 0:
                                host_out[s + off:s + off + cnt].copy_(final[s + off:s + off + cnt], non_blocking=True)
                else:
                    for (s, e) in bounds:
                        cnt = max(0, min(ln, (e - s) - off))
                        if cnt > 0:
                            host_out[s + off:s + off + cnt].copy_(final[s + off:s + off + cnt])
        if use_streams:
            torch.cuda.current_stream(dev).wait_stream(comm)
            if d2h is not None:
                d2h.synchronize()
        return final
