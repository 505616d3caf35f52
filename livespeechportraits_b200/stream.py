"""Live audio through demo.py stages 1-4: samples pushed in pieces of any size come out as mouth and head-pose track rows
as soon as the models allow, bit-identical to the whole-clip calls on the concatenated audio.

Each stage has a stream object (``MelFrontEnd.stream``, ``ApcEncoder.stream``, ``MouthGenerator.stream``,
``HeadposeGenerator.stream``) that carries its state between pushes on the device; ``AudioStream`` chains them, with the
manifold projection (row by row, so it needs no state) in between.  Which rows a push may return is a pure function of
the samples pushed so far and of whether the stream has finished (``ready_counts``), computed on the host, so a push
never waits for the device.

The look-ahead is the models': Audio2Mouth's ``frame_future`` (18) and Audio2Headpose's (15) video frames, i.e. about
0.32 s and 0.27 s of audio at 60 fps, plus the mel window itself.

``PortraitStream`` goes on to frames: the track rows through stage 5 (``LandmarkPostprocessor.stream``, which adds the
smoothing radii to the look-ahead: frame t needs head-pose row t + max(rr, rt), so for May's settings APC pair t + 55),
then the rasteriser and the generator, one frame per generator call.

Both streams take 16 kHz mono samples, or native-rate frames through an ``audio.Resampler`` (``AudioStream(...,
resampler=...)``): librosa.load's mono mix and resampling, streamed bit for bit, with ``resample_counts`` frames of
look-ahead in front (about 4 ms at 48 kHz).
"""
from __future__ import annotations

import dataclasses
import math
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


def resample_counts(n_in: int, finished: bool, orig_sr: int, res_type: str = "kaiser_best", sr: int = SR) -> int:
    """16 kHz samples ready after ``n_in`` native-rate frames (``audio.ResampleStream``).  Output t reads input frames
    up to n + nwin // index_step, n = int(register(t)) (the right wing's longest reach), so it is ready once those are
    in and t < int(n_in * ratio) (resampy's count, monotone in n_in).  At the end of the clip all ``ceil(n_in * ratio)``
    (``fix_length``'s zero included), or 0 where resampy refuses the clip.  At ``orig_sr == sr`` every frame, at once."""
    if orig_sr == sr:
        return n_in
    from .audio import filter_shape, register_at, register_table
    ratio = float(sr) / orig_sr
    total = int(n_in * ratio)
    if finished:
        return int(math.ceil(n_in * ratio)) if total >= 1 else 0
    nwin, _, index_step = filter_shape(orig_sr, res_type, sr)
    last = n_in - 1 - nwin // index_step                 # the last frame an output may read from its window's centre
    if last < 0:
        return 0
    reg = register_table(ratio)
    t = max(0, int(last * ratio))                        # near the count; the fp64 registers decide
    while t > 0 and int(register_at(reg, t - 1)) > last:
        t -= 1
    while int(register_at(reg, t)) <= last:
        t += 1
    return min(t, total)


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


def landmark_counts(n_feat: int, n_head: int, finished: bool, rm: int, rh: int) -> int:
    """Stage-5 frames ready from ``n_feat`` mouth and ``n_head`` head-pose track rows: frame t needs mouth rows up to
    t + rm (and t + rm < n_head, since the mouth reflects at nframe = min(n_feat, n_head)) and head rows up to t + rh;
    at the end of the clip all ``min(n_feat, n_head)`` frames."""
    if finished:
        return min(n_feat, n_head)
    return max(0, min(min(n_feat, n_head) - rm, n_head - rh))


def portrait_counts(n_samples: int, finished: bool, params, frame_len: int = 266, step: float = SR * 0.5 / FPS,
                    mouth_future: int = 18, headpose_future: int = 15) -> int:
    """Portrait frames ready after ``n_samples`` samples: ``landmark_counts`` of the track rows ``ready_counts`` gives,
    with the radii of ``params`` (``landmarks.StageParams``)."""
    from .landmarks import radii
    c = ready_counts(n_samples, finished, frame_len, step, mouth_future, headpose_future)
    return landmark_counts(c.mouth, c.headpose, finished, *radii(params))


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
    projector), bit for bit.  With ``resampler`` (an ``audio.Resampler``) ``push`` takes native-rate frames and the
    audio is ``resampler.resample`` of them, streamed (``ResampleStream``); the counts are then ``ready_counts`` of
    ``resample_counts``.  ``noise`` is as for ``HeadposeGenerator.stream``: None draws from torch's global CPU
    generator frame by frame, in the order the whole-clip draw takes.

    Device memory does not grow with the stream: the audio tail of the next window, one APC row waiting for its pair, the
    last APC row, the head-pose rows not consumed yet, the fixed-size recurrent states and the stages' workspaces, which
    are allocated for the largest push so far and reused, so pushes of one size allocate nothing that outlives them.
    All pushes of a session go on one CUDA stream (the current one when ``push`` is called)."""

    def __init__(self, mel, apc, mouth, headpose, projector=None, k: int = 10, percent: float = 1.0, pre_headpose=None,
                 sigma_scale: float = 0.3, noise=None, winlen: float = 1 / 60, winstep: float = 0.5 / 60, sr: int = SR,
                 resampler=None):
        self._rs = resampler.stream() if resampler is not None else None
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
        if self._rs is not None:
            samples = self._rs.push(samples)
        return self._step(self._mel.push(samples), False)

    def finish(self) -> StreamRows:
        if self.finished:
            raise RuntimeError("the stream has finished")
        self.finished = True
        if self._rs is not None:
            return self._step(torch.cat([self._mel.push(self._rs.finish()), self._mel.finish()]), True)
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


@dataclasses.dataclass
class PortraitFrames:
    """What one ``PortraitStream.push`` or ``finish`` returned: frames ``frame0 .. frame0 + k - 1``."""
    frames: torch.Tensor          # [k, H, W, 3] uint8 images (tensor2im's layout)
    frame0: int
    landmarks: torch.Tensor       # [k, 73, 2] the landmarks they were drawn from
    shoulders: torch.Tensor       # [k, 18, 2]
    rows: StreamRows              # the track rows of stages 1-4 this push produced


class PortraitStream:
    """Live audio to portrait frames: ``AudioStream`` (stages 1-4) -> ``LandmarkStream`` (stage 5) ->
    ``net.draw_feature_maps`` -> ``net.render_image`` (stage 6).  ``push(samples)`` / ``finish()`` return
    ``PortraitFrames``; how many is ``portrait_counts`` (of ``resample_counts`` when the audio stream resamples).

    ``audio_stream`` is a fresh ``AudioStream``; ``post`` a ``LandmarkPostprocessor``, ``params`` its ``StageParams``;
    ``net`` the ``Feature2Face_G`` and ``cand`` its candidate images ``[1, 3 k, H, W]`` on the device.  The landmarks
    follow ``LandmarkStream``'s live lip-fix rule.  A push's feature maps are rasterised in one call into a staging
    buffer kept across pushes (the rasteriser is exact frame by frame); the generator then renders one frame per call,
    so every frame goes through the same plan and the same CUDA graph and its bits do not depend on the push sizes.
    Pushes make no host synchronisation and go on one CUDA stream."""

    def __init__(self, audio_stream: AudioStream, post, params, net, cand, size=(512, 512), image_pad=None):
        self._audio = audio_stream
        self._lm = post.stream(params, image_pad)
        self._net, self._cand = net, cand
        self._size = (int(size[0]), int(size[1]))
        self._maps = None                     # [k, 1, H, W] staging for the feature maps, kept across pushes
        self.frames = 0

    def push(self, samples) -> PortraitFrames:
        rows = self._audio.push(samples)
        return self._render(rows, [self._lm.push(rows.mouth, rows.headpose)])

    def finish(self) -> PortraitFrames:
        rows = self._audio.finish()
        return self._render(rows, [self._lm.push(rows.mouth, rows.headpose), self._lm.finish()])

    def _render(self, rows: StreamRows, parts) -> PortraitFrames:
        lm = torch.cat([p.landmarks for p in parts]) if len(parts) > 1 else parts[0].landmarks
        sh = torch.cat([p.shoulders for p in parts]) if len(parts) > 1 else parts[0].shoulders
        k = lm.shape[0]
        w, h = self._size
        if self._maps is None or self._maps.shape[0] < k:
            self._maps = torch.empty((max(k, 1), 1, h, w), dtype=torch.float32, device=lm.device)
        frames = torch.empty((k, h, w, 3), dtype=torch.uint8, device=lm.device)
        if k:
            maps = self._net.draw_feature_maps(lm, sh, self._size, out=self._maps[:k])
            for i in range(k):
                self._net.render_image(maps[i:i + 1], self._cand, out=frames[i:i + 1])
        out = PortraitFrames(frames, self.frames, lm, sh, rows)
        self.frames += k
        return out
