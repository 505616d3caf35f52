"""Streaming without a GPU: the emission arithmetic of livespeechportraits_b200/stream.py, AudioStream's chunking driven by
float64 host stand-ins of the stages (restatements of the oracle emulators with carried state), and the argument checks
of the stream entry points of the C ABIs on host-only handles."""
import ctypes as C

import numpy as np
import pytest
import torch

from livespeechportraits_b200 import _lib, headpose
from livespeechportraits_b200.stream import AudioStream, mel_windows, ready_counts
from oracle import a2h_oracle as A
from oracle import rnn_oracle as R
from a2h_incremental import generate_incremental, lrelu

STEP, FRAME = 16000 * 0.5 / 60, 266
N_WAV = 183_296                                         # 00083.wav


# ----------------------------------------------------------------------------------------------------------------------
# Emission counts
# ----------------------------------------------------------------------------------------------------------------------
def _whole_shapes(n):
    mel = 2 * int(n / 16000 * 60)
    return mel, mel, mel // 2, max(0, mel // 2 - 15)


def test_totals_at_finish_are_the_whole_clip_shapes():
    for n in list(range(0, 20001)) + [N_WAV]:
        assert tuple(ready_counts(n, True)) == _whole_shapes(n), n


def test_counts_are_monotone_and_need_only_pushed_samples():
    prev = ready_counts(0, False)
    for n in range(0, 20001):
        c = ready_counts(n, False)
        assert all(a <= b for a, b in zip(prev, c)) and all(a <= b for a, b in zip(c, ready_counts(n, True))), n
        if c.mel:
            assert int((c.mel - 1) * STEP) + FRAME <= n                  # the last ready window has all its samples
        assert c.apc == c.mel and c.mouth <= max(0, c.apc // 2 - 18)      # mouth frame f needs APC pair f + 18
        assert c.headpose <= max(0, c.apc // 2 - 15)                      # head-pose frame i needs pair i + 15
        prev = c


def test_a_row_is_ready_on_the_sample_that_completes_it():
    for i in (0, 1, 2, 5, 100, 1373):
        end = int(i * STEP) + FRAME                                      # samples window i needs
        end = max(end, int(np.ceil((i // 2 + 1) * 16000 / 60)))          # and the clip count that includes it
        while 2 * int(end / 16000 * 60) <= i:
            end += 1
        assert mel_windows(end - 1, False) == i and mel_windows(end, False) == i + 1, i
    # mouth frame 0 waits for APC pair 18 (rows 36, 37), head-pose frame 0 for pair 15
    for stage, pair in (("mouth", 18), ("headpose", 15)):
        n = next(n for n in range(30000) if ready_counts(n, False).apc >= 2 * pair + 2)
        assert getattr(ready_counts(n - 1, False), stage) == 0 and getattr(ready_counts(n, False), stage) == 1


# ----------------------------------------------------------------------------------------------------------------------
# Host stand-ins of the stages, with carried state
# ----------------------------------------------------------------------------------------------------------------------
class MelStandIn:
    """Window i -> 4 statistics of its zero-padded clip (fp32 values in float64); keeps every sample pushed."""

    def stream(self, winlen, winstep, sr):
        return self

    def __init__(self):
        self.audio, self.done, self.n = np.zeros(0), 0, 0

    @staticmethod
    def window(audio, i):
        st = int(i * STEP)
        c = np.zeros(FRAME)
        seg = audio[st:st + FRAME]
        c[:seg.shape[0]] = seg
        return np.array([c.sum(), (c * c).sum(), c[0], c[-1]], np.float32).astype(np.float64)   # fp32 values, as mel frames

    def whole(self, audio):
        return np.array([self.window(audio, i) for i in range(2 * int(len(audio) / 16000 * 60))]).reshape(-1, 4)

    def _emit(self, finished):
        ready = mel_windows(self.n, finished)
        out = np.array([self.window(self.audio, i) for i in range(self.done, ready)]).reshape(-1, 4)
        self.done = ready
        return torch.from_numpy(out)

    def push(self, samples):
        self.audio = np.concatenate([self.audio, np.asarray(samples, np.float64)])
        self.n += len(samples)
        return self._emit(False)

    def finish(self):
        return self._emit(True)


def _rnn_steps(x, w_ih, b, w_hh, b_hn, G, H, h, c):
    """rnn_oracle._rnn_emulate (cl = 1) from state (h, c), input projection row by row; returns (out, h, c)."""
    out = np.empty((x.shape[0], H))
    for t in range(x.shape[0]):
        xg = (w_ih.reshape(G * H, -1) @ x[t] + b).reshape(H, G)
        gh = (w_hh.reshape(G * H, H) @ h).reshape(H, G)
        if G == 3:
            r = 1 / (1 + np.exp(-(xg[:, 0] + gh[:, 0])))
            z = 1 / (1 + np.exp(-(xg[:, 1] + gh[:, 1])))
            n = np.tanh(xg[:, 2] + r * (gh[:, 2] + b_hn))
            h = n + z * (h - n)
        else:
            i = 1 / (1 + np.exp(-(xg[:, 0] + gh[:, 0])))
            f = 1 / (1 + np.exp(-(xg[:, 1] + gh[:, 1])))
            g = np.tanh(xg[:, 2] + gh[:, 2])
            o = 1 / (1 + np.exp(-(xg[:, 3] + gh[:, 3])))
            c = f * c + i * g
            h = o * np.tanh(c)
        out[t] = h
    return out, h, c


class ApcStandIn:
    """emulate_apc's GRU stack (2 layers, 16 units) with each layer's h carried between pushes."""
    H, L = 16, 2

    def __init__(self, seed=0):
        rng = np.random.default_rng(seed)
        self.arrays = {}
        for l in range(self.L):
            In = 4 if l == 0 else self.H
            for j, shape in enumerate([(3 * self.H * In,), (3 * self.H,), (3 * self.H * self.H,), (self.H,)]):
                self.arrays[4 * l + j] = rng.uniform(-0.4, 0.4, shape)

    def stream(self):
        self.h = [np.zeros(self.H) for _ in range(self.L)]
        return self

    def push(self, mel):
        x = mel.numpy()
        for l in range(self.L):
            a = [self.arrays[4 * l + j] for j in range(4)]
            x, self.h[l], _ = _rnn_steps(x, a[0], a[1], a[2], a[3], 3, self.H, self.h[l], None)
        return torch.from_numpy(x.reshape(-1, self.H))

    def finish(self):
        return torch.zeros((0, self.H), dtype=torch.float64)


class MouthStandIn:
    """Audio2Mouth's shape with small widths: downsample over pairs, one LSTM layer carried between pushes, fc on the steps
    >= frame_future; finish() feeds 2 frame_future copies of the last row."""
    H, OUT = 8, 3

    def __init__(self, ff, D=16, seed=1):
        rng = np.random.default_rng(seed)
        self.ff, self.D = ff, D
        self.w_ds = rng.uniform(-0.3, 0.3, (D, 2 * D))
        self.lstm = [rng.uniform(-0.4, 0.4, s) for s in [(4 * self.H * D,), (4 * self.H,), (4 * self.H * self.H,)]]
        self.w_fc = rng.uniform(-0.5, 0.5, (self.OUT, self.H))

    def stream(self):
        self.h, self.c, self.pairs, self.odd, self.last = np.zeros(self.H), np.zeros(self.H), 0, None, None
        return self

    def _run(self, x):
        ds = np.array([lrelu(self.w_ds @ x[2 * p:2 * p + 2].reshape(-1)) for p in range(x.shape[0] // 2)]).reshape(-1, self.D)
        y, self.h, self.c = _rnn_steps(ds, *self.lstm, None, 4, self.H, self.h, self.c)
        keep = np.arange(self.pairs, self.pairs + y.shape[0]) >= self.ff
        self.pairs += y.shape[0]
        return torch.from_numpy(np.array([self.w_fc @ r for r in y[keep]]).reshape(-1, self.OUT))

    def push(self, feats):
        x = feats.numpy()
        assert x.shape[0] % 2 == 0                       # AudioStream hands over whole pairs only
        if x.shape[0]:
            self.last = x[-1]
        return self._run(x)

    def finish(self):
        if not self.pairs:
            return torch.zeros((0, self.OUT), dtype=torch.float64)
        return self._run(np.repeat(self.last[None], 2 * self.ff, axis=0))

    def whole(self, feats):
        self.stream()
        x = np.concatenate([feats, np.repeat(feats[-1:], 2 * self.ff, axis=0)])
        return self._run(x).numpy()


class HeadposeStandIn:
    """tests/a2h_incremental.generate_incremental with its history as a ring of 128 steps and the last sample carried
    between pushes; audio_downsample and the conditioning projections row by row, as they arrive."""

    def __init__(self, opt, sd):
        self.opt, self.sd = opt, sd
        f64 = lambda k: sd[k].double().numpy()      # noqa: E731
        self.dil, self.rf, self.ff = A.dilations(opt), opt.A2H_receptive_field, opt.frame_future
        self.ring = 128
        nl = len(self.dil)
        self.Wc = [(f64(f"WaveNet.residual_blocks.{i}.cond_filter_conv.weight")[:, :, 0], f64(f"WaveNet.residual_blocks.{i}.cond_filter_conv.bias"),
                    f64(f"WaveNet.residual_blocks.{i}.cond_gate_conv.weight")[:, :, 0], f64(f"WaveNet.residual_blocks.{i}.cond_gate_conv.bias"))
                   for i in range(nl)]
        self.W1, self.b1 = f64("WaveNet.start_conv1.weight")[:, :, 0], f64("WaveNet.start_conv1.bias")
        self.W2, self.b2 = f64("WaveNet.start_conv2.weight")[:, :, 0], f64("WaveNet.start_conv2.bias")
        self.E1, self.e1 = f64("WaveNet.end_conv_1.weight")[:, :, 0], f64("WaveNet.end_conv_1.bias")
        self.E2, self.e2 = f64("WaveNet.end_conv_2.weight")[:, :, 0], f64("WaveNet.end_conv_2.bias")
        self.blk = []
        for i in range(nl):
            p = f"WaveNet.residual_blocks.{i}."
            self.blk.append(dict(Wf=f64(p + "filter_conv.weight"), bf=f64(p + "filter_conv.bias"), Wg=f64(p + "gate_conv.weight"),
                                 bg=f64(p + "gate_conv.bias"), Wr=f64(p + "residual_conv.weight")[:, :, 0],
                                 br=f64(p + "residual_conv.bias"), Ws=f64(p + "skip_conv.weight")[:, :, 0], bs=f64(p + "skip_conv.bias")))
        self.ds_sd = {k: v.double() for k, v in sd.items() if k.startswith("audio_downsample") and v.dtype.is_floating_point}

    def stream(self, pre_headpose, sigma_scale, noise):
        self.h = np.zeros(self.opt.A2H_GMM_ndim) if pre_headpose is None else np.asarray(pre_headpose, np.float64)
        self.sigma, self.noise = sigma_scale, noise
        self.X = np.zeros((len(self.dil), self.ring, self.opt.A2H_wavenet_residual_channels))
        self.cond, self.rows, self.frames = {}, 0, 0                # cond of the rows not consumed yet, by absolute row
        return self

    def _cond(self, row):
        with torch.no_grad():
            ds = A.audio_downsample(self.ds_sd, torch.from_numpy(row[None])).numpy()[0]
        return [(wf @ ds + bf, wg @ ds + bg) for wf, bf, wg, bg in self.Wc]

    def _step(self, t, emit_row):
        r = max(t + self.ff - (self.rf - 1), 0)
        x = lrelu(self.W2 @ lrelu(self.W1 @ self.h + self.b1) + self.b2)
        skip = 0.0
        for l, d in enumerate(self.dil):
            self.X[l, t % self.ring] = x
            xd = self.X[l, (t - d) % self.ring] if t - d >= 0 else np.zeros_like(x)
            B, (cf, cg) = self.blk[l], self.cond[r][l]
            f = B["Wf"][:, :, 0] @ xd + B["Wf"][:, :, 1] @ x + B["bf"] + cf
            g = B["Wg"][:, :, 0] @ xd + B["Wg"][:, :, 1] @ x + B["bg"] + cg
            z = np.tanh(f) * (1.0 / (1.0 + np.exp(-g)))
            skip = skip + B["Ws"] @ z + B["bs"]
            x = B["Wr"] @ z + B["br"] + x
        if emit_row is None:
            return None
        out = self.E2 @ lrelu(self.E1 @ lrelu(skip) + self.e1) + self.e2
        nd = self.opt.A2H_GMM_ndim
        self.h = emit_row * (np.exp(-out[1 + nd:1 + 2 * nd]) * self.sigma) + out[1:1 + nd]
        return self.h

    def push(self, rows):
        rows = rows.numpy()
        for j in range(rows.shape[0]):
            self.cond[self.rows + j] = self._cond(rows[j])
        self.rows += rows.shape[0]
        n = max(0, self.rows - self.ff) - self.frames
        noise = self.noise(self.frames, n) if n else None
        out = []
        for j in range(n):
            i = self.frames + j
            steps = range(self.rf - 1) if i == 0 else ()
            for t in steps:                                          # frame 0 first replays window 0
                self._step(t, None)
            out.append(self._step(i + self.rf - 1, np.asarray(noise[j], np.float64)).copy())
        self.frames += n
        for r in [r for r in self.cond if r < self.frames + self.ff and self.frames]:
            del self.cond[r]                                          # rows no later frame reads
        assert len(self.cond) <= self.ff + 1
        return torch.from_numpy(np.array(out).reshape(-1, self.opt.A2H_GMM_ndim))

    def finish(self):
        return torch.zeros((0, self.opt.A2H_GMM_ndim), dtype=torch.float64)


def _stand_ins(mouth_ff=18):
    opt = A.default_opt(APC_hidden_size=16, A2H_wavenet_cond_channels=16)
    sd = A.make_state_dict(opt, "B", 1)
    return MelStandIn(), ApcStandIn(), MouthStandIn(mouth_ff), HeadposeStandIn(opt, sd), opt, sd


def _run(audio, sizes, mouth_ff=18):
    mel, apc, mouth, head, opt, sd = _stand_ins(mouth_ff)
    noise = A.reference_noise(4000, 12, 1, seed=3).astype(np.float64)
    s = AudioStream(mel, apc, mouth, head, pre_headpose=np.zeros(12), sigma_scale=0.3, noise=lambda i0, n: noise[i0:i0 + n])
    outs, at = [], 0
    for k in sizes:
        outs.append(s.push(audio[at:at + k]))
        at = min(at + k, len(audio))
        c = ready_counts(at, False, mouth_future=mouth_ff)
        assert (s.apc_rows, s.mouth_frames, s.headpose_frames) == (c.apc, c.mouth, c.headpose)
    outs.append(s.finish())
    cat = lambda key: torch.cat([getattr(o, key) for o in outs]).numpy()          # noqa: E731
    return cat("apc"), cat("mouth"), cat("headpose"), (mel, apc, mouth, head, opt, sd, noise)


def _sizes(n, seed):
    rng = np.random.default_rng(seed)
    out = [0, 1, 0, 1]
    while sum(out) < n:
        out.append(int(rng.choice([0, 1, 2, 133, 267, 400, 1999])))
    return out


@pytest.mark.parametrize("n,mouth_ff", [(183_296 // 8, 18), (4800, 18), (4000, 0), (1400, 18), (0, 18)])
def test_session_chunks_give_the_whole_clip_rows(n, mouth_ff):
    """Pushes of 0 and 1 samples, odd APC rows split across pushes, a stream shorter than frame_future (1400 samples:
    5 pairs), and a head-pose stream of about 170 frames, past the 128-step ring."""
    audio = np.random.default_rng(n).uniform(-0.5, 0.5, n)
    apc, mouth, head, (mel_s, apc_s, mouth_s, head_s, opt, sd, noise) = _run(audio, _sizes(n, n + 1), mouth_ff)
    whole_mel = mel_s.whole(audio)
    whole_apc = apc_s.stream().push(torch.from_numpy(whole_mel)).numpy()
    assert np.array_equal(apc, whole_apc)
    packed = lambda w: apc_s.arrays[w]                                             # noqa: E731
    assert np.allclose(apc, R.emulate_apc(packed, whole_mel, 2, cl=1, hidden=16), rtol=0, atol=1e-12)
    if whole_apc.shape[0]:
        assert np.array_equal(mouth, mouth_s.whole(whole_apc))
    assert mouth.shape[0] == whole_apc.shape[0] // 2
    pairs = whole_apc.reshape(-1, 32)
    nframe = pairs.shape[0] - 15
    if nframe > 0:
        whole_head = HeadposeStandIn(opt, sd).stream(np.zeros(12), 0.3, lambda i0, k: noise[i0:i0 + k]).push(torch.from_numpy(pairs))
        assert np.array_equal(head, whole_head.numpy())
        ref = generate_incremental(sd, pairs, np.zeros(12), noise[:nframe], opt, 0.3)
        assert np.allclose(head, ref, rtol=0, atol=1e-9)
    assert head.shape[0] == max(0, nframe)


# ----------------------------------------------------------------------------------------------------------------------
# ABI checks on host-only handles
# ----------------------------------------------------------------------------------------------------------------------
ENODEV, EINVAL = -2, -1


def _handles(lib):
    hs = {}
    for prefix, args in (("lspa", ()), ("lsph", (C.byref(headpose.config_from_opt(A.default_opt())),))):
        h = C.c_void_p()
        assert getattr(lib, prefix + "_create")(C.byref(h), *args, -1) == 0
        hs[prefix] = h
    for kind, cfg in (("apc", (80, 512, 3, 0, 0, 0)), ("mouth", (512, 0, 0, 0, 18, 75))):
        c = _lib.LsprConfig(_lib.LSPR_KIND[kind], *cfg)
        h = C.c_void_p()
        assert lib.lspr_create(C.byref(h), C.byref(c), -1) == 0
        hs[kind] = h
    return hs


def test_stream_symbols_are_bound():
    for name in ("lspa_logmel_at", "lspr_state_bytes", "lspr_forward_stream", "lsph_state_bytes",
                 "lsph_stream_workspace_bytes", "lsph_generate_stream"):
        assert name in _lib.ARGTYPES
        assert getattr(_lib.load(), name).argtypes == _lib.ARGTYPES[name]
    # a whole clip is the span from 0: the library exports no second entry point for it, so a caller of the old
    # whole-clip signatures fails at symbol lookup instead of passing the wrong arguments
    for name in ("lspa_logmel", "lspr_forward", "lsph_generate"):
        assert name not in _lib.ARGTYPES
        assert not hasattr(_lib.load(), name)


def test_stream_calls_on_host_only_handles():
    lib = _lib.load()
    hs = _handles(lib)
    P = 1 << 12                                                   # a 256-byte aligned stand-in pointer (never read)
    sz = C.c_size_t()
    try:
        assert lib.lspr_state_bytes(hs["apc"], C.byref(sz)) == 0 and sz.value == 4 * 3 * 2 * 512
        assert lib.lspr_state_bytes(hs["mouth"], C.byref(sz)) == 0 and sz.value == 4 * 3 * 2 * 256
        assert lib.lsph_state_bytes(hs["lsph"], C.byref(sz)) == 0 and sz.value == 4 * (14 * 128 * 128 + 32)
        assert lib.lsph_stream_workspace_bytes(hs["lsph"], 3, C.byref(sz)) == 0 and sz.value > 0
        ws = sz.value
        # mel: a window that starts before the first sample given; ENODEV otherwise
        assert lib.lspa_logmel_at(hs["lspa"], P, 134, 400, 1, 1, 266, STEP, 1, P, None) == EINVAL      # window 1 starts at 133
        assert b"before the first sample" in lib.lspa_last_error()
        assert lib.lspa_logmel_at(hs["lspa"], P, 133, 400, 1, 1, 266, STEP, 1, P, None) == ENODEV
        # recurrent: null state, odd Audio2Mouth row count; ENODEV otherwise
        assert lib.lspr_forward_stream(hs["apc"], P, 4, 0, P, None, P, 1 << 30, 0, None) == EINVAL
        assert b"null state" in lib.lspr_last_error()
        assert lib.lspr_forward_stream(hs["mouth"], P, 3, 0, P, P, P, 1 << 30, 0, None) == EINVAL
        assert b"even" in lib.lspr_last_error()
        assert lib.lspr_forward_stream(hs["apc"], P, 4, 7, P, P, P, 1 << 30, 0, None) == ENODEV
        assert lib.lspr_forward_stream(hs["mouth"], P, 4, 7, P, P, P, 1 << 30, 0, None) == ENODEV
        # head pose: frames 10 .. 12 need audio rows 25 .. 27; frame 0 needs rows from 0
        gen = lib.lsph_generate_stream
        assert gen(hs["lsph"], P, 25, 3, 10, 3, P, P, None, 0.3, P, None, None, P, ws, 0, None) == EINVAL
        assert b"null state" in lib.lsph_last_error()
        assert gen(hs["lsph"], P, 26, 3, 10, 3, P, P, None, 0.3, P, None, P, P, ws, 0, None) == EINVAL
        assert gen(hs["lsph"], P, 25, 2, 10, 3, P, P, None, 0.3, P, None, P, P, ws, 0, None) == EINVAL
        assert b"need audio rows 25 .. 27" in lib.lsph_last_error()
        assert gen(hs["lsph"], P, 15, 3, 0, 3, P, P, None, 0.3, P, None, P, P, ws, 0, None) == EINVAL
        assert gen(hs["lsph"], P, 25, 3, 10, 3, P, P, None, 0.3, P, None, P, P, ws, 0, None) == ENODEV
    finally:
        for k, h in hs.items():
            getattr(lib, ("lspr" if k in ("apc", "mouth") else k) + "_destroy")(h)
