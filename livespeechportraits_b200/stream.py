"""Live audio through demo.py stages 1-4: samples pushed in pieces of any size come out as mouth and head-pose track rows
as soon as the models allow, bit-identical to the whole-clip calls on the concatenated audio.

Each stage has a stream object (``MelFrontEnd.stream``, ``ApcEncoder.stream``, ``MouthGenerator.stream``,
``HeadposeGenerator.stream``) that carries its state between pushes on the device; ``AudioStream`` chains them, with the
manifold projection (row by row, so it needs no state) in between.  Which rows a push may return is a pure function of
the samples pushed so far and of whether the stream has finished (``ready_counts``), computed on the host, so a push
never waits for the device.

The look-ahead is the models': Audio2Mouth's ``frame_future`` (18) and Audio2Headpose's (15) video frames, i.e. about
0.32 s and 0.27 s of audio at 60 fps, plus the mel window itself.
"""
from __future__ import annotations

import dataclasses
from typing import NamedTuple, Optional

import torch

from . import _lib

SR = 16000
FPS = 60


def mel_windows(n_samples: int, finished: bool, frame_len: int = 266, step: float = SR * 0.5 / FPS) -> int:
    """Windows ready after ``n_samples`` samples: every i < ``2 int(n / 16000 * 60)`` (funcs/utils.py:67, the final count
    of ``MelFrontEnd.logmel``) whose ``frame_len`` samples from ``int(i * step)`` are all in; at the end of the clip all
    of them (the last ones read the zero end padding)."""
    total = 2 * int(n_samples / 16000 * 60)
    if finished:
        return total
    i = max(0, int((n_samples - frame_len) / step))      # near the count of windows that fit; the fp64 starts decide
    while i > 0 and int((i - 1) * step) + frame_len > n_samples:
        i -= 1
    while int(i * step) + frame_len <= n_samples:
        i += 1
    return min(i, total)


class Counts(NamedTuple):
    mel: int          # log-mel windows = APC rows
    apc: int
    mouth: int        # Audio2Mouth track rows
    headpose: int     # head-pose track rows


def ready_counts(n_samples: int, finished: bool, frame_len: int = 266, step: float = SR * 0.5 / FPS,
                 mouth_future: int = 18, headpose_future: int = 15) -> Counts:
    """Rows of each stage ready after ``n_samples`` samples (``finished``: the clip has ended).  An APC row needs its mel
    window; a video frame is a pair of APC rows; mouth frame f needs pair f + mouth_future (at the end the missing pairs
    are copies of the last APC row); head-pose frame i needs pair i + headpose_future (no end padding).  At the end the
    totals are the whole-clip shapes: 2 nframe, 2 nframe, nframe, nframe - headpose_future (or 0)."""
    mel = mel_windows(n_samples, finished, frame_len, step)
    pairs = mel // 2
    mouth = pairs if finished else max(0, pairs - mouth_future)
    return Counts(mel, mel, mouth, max(0, pairs - headpose_future))


@dataclasses.dataclass
class StreamRows:
    """What one ``push`` or ``finish`` returned: the new rows of each stage and the clip index of their first row."""
    mouth: torch.Tensor           # [m, out_dim] Audio2Mouth track rows
    mouth_frame0: int
    headpose: torch.Tensor        # [h, ndim] head-pose track rows
    headpose_frame0: int
    apc: torch.Tensor             # [a, APC_hidden] APC features
    features: torch.Tensor        # [a, APC_hidden] the rows fed to the two generators (blended when projecting)
    apc_row0: int


class AudioStream:
    """Stages 1-4 of demo.py over live audio: ``push(samples)`` (16 kHz mono; any count, 0 included) and ``finish()``
    return ``StreamRows``.  The concatenated tracks equal ``mouth.generate(blend)`` and
    ``headpose.generate(blend.view(-1, 2 * APC_hidden), pre_headpose, noise, sigma_scale)`` of the whole clip, with
    ``blend = projector.project_features(apc.forward(mel.logmel(audio)), k, percent)`` (or the APC features without a
    projector), bit for bit.  ``noise`` is as for ``HeadposeGenerator.stream``: None draws from torch's global CPU
    generator frame by frame, in the order the whole-clip draw takes.

    Device memory does not grow with the stream: the audio tail of the next window, one APC row waiting for its pair, the
    last APC row, the head-pose rows not consumed yet, the fixed-size recurrent states and the stages' workspaces, which
    are allocated for the largest push so far and reused, so pushes of one size allocate nothing that outlives them.
    All pushes of a session go on one CUDA stream (the current one when ``push`` is called)."""

    def __init__(self, mel, apc, mouth, headpose, projector=None, k: int = 10, percent: float = 1.0, pre_headpose=None,
                 sigma_scale: float = 0.3, noise=None, winlen: float = 1 / 60, winstep: float = 0.5 / 60, sr: int = SR):
        self._mel = mel.stream(winlen, winstep, sr)
        self._apc = apc.stream()
        self._mouth = mouth.stream()
        self._head = headpose.stream(pre_headpose, sigma_scale, noise)
        self._proj, self._k, self._percent = projector, int(k), float(percent)
        self._odd = None                       # a feature row waiting for its pair
        self._proj_ws = None                   # the projection's workspace, kept across pushes
        self.apc_rows = self.mouth_frames = self.headpose_frames = 0
        self.finished = False

    def push(self, samples) -> StreamRows:
        if self.finished:
            raise RuntimeError("the stream has finished")
        return self._step(self._mel.push(samples), False)

    def finish(self) -> StreamRows:
        if self.finished:
            raise RuntimeError("the stream has finished")
        self.finished = True
        return self._step(self._mel.finish(), True)

    def _step(self, mel: torch.Tensor, finished: bool) -> StreamRows:
        apc = self._apc.push(mel)
        if finished:
            apc = torch.cat([apc, self._apc.finish()])
        feats = apc
        if self._proj is not None and apc.shape[0]:
            self._proj_ws = _lib.reserve(self._proj_ws, self._proj.workspace_bytes(apc.shape[0], self._k), apc.device)
            feats = self._proj.project_features(apc, self._k, self._percent, ws=self._proj_ws)
        rows = torch.cat([self._odd, feats]) if self._odd is not None else feats
        even = rows.shape[0] // 2 * 2
        self._odd = rows[even:].clone() if even < rows.shape[0] else None
        pairs = rows[:even]
        mouth = self._mouth.push(pairs)
        head = self._head.push(pairs.reshape(-1, 2 * pairs.shape[1]))
        if finished:
            mouth = torch.cat([mouth, self._mouth.finish()])
            head = torch.cat([head, self._head.finish()])
        out = StreamRows(mouth, self.mouth_frames, head, self.headpose_frames, apc, feats, self.apc_rows)
        self.apc_rows += apc.shape[0]
        self.mouth_frames += mouth.shape[0]
        self.headpose_frames += head.shape[0]
        return out
