"""Live stage 5 and live portraits on the host: the emission counts of ``stream.landmark_counts`` /
``stream.portrait_counts`` against their brute-force definitions; the live lip-fix truth (``live_truth``) against
``landmark_oracle.truth`` on the landmark goldens, and every planted defect of the live path caught by the bound;
``LandmarkStream`` and ``PortraitStream`` bookkeeping driven by float64 stand-ins; the argument checks of
``lspl_run_stream`` on host-only handles."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

import live_landmark_oracle as L
from livespeechportraits_b200 import _lib
from livespeechportraits_b200.landmarks import LandmarkStream, StageParams, radii
from livespeechportraits_b200.stream import AudioStream, PortraitStream, landmark_counts, portrait_counts, ready_counts
from oracle import landmark_oracle as O

GOLD_DIR = os.path.join(os.path.dirname(__file__), "golden", "landmarks")
GOLDENS = ["may_672", "obama1_672", "xy_200", "lowermore_200", "mouth_sigma0_150", "head_longer_300_340",
           "feat_longer_340_300", "no_crossing_200", "n1", "n2", "n7", "n41", "pad_200"]
KEYS = ("landmarks", "shoulders", "final_pts3d", "pred_headpose")


def _golden(name):
    g = np.load(os.path.join(GOLD_DIR, name + ".npz"))
    ident = {k: g["id_" + k] for k in O.IDENTITY_KEYS}
    ident["scale"] = np.float64(ident["scale"])
    pad = tuple(int(v) for v in g["image_pad"]) or None
    return g["pred_Feat"], g["pred_Head"], ident, json.loads(str(g["params"])), pad


def _stage_params(prm):
    return StageParams(prm["Feat_smooth_sigma"], prm["AMP_method"], prm["Feat_AMPs"], prm["rot_AMP"], prm["trans_AMP"],
                       prm["Head_smooth_sigma"], prm["shoulder_AMP"])


# ----------------------------------------------------------------------------------------------------------------------
# emission counts
# ----------------------------------------------------------------------------------------------------------------------
def _brute(F, H, finished, rm, rh):
    """Frame t is out when its windows are interior: t + rm < min(F, H) and t + rh < H; at the end every t < min(F, H)."""
    n = 0
    while n < min(F, H) and (finished or (n + rm < min(F, H) and n + rh < H)):
        n += 1
    return n


def test_landmark_counts_match_the_definition():
    t = np.arange(201)
    F, H = np.meshgrid(np.arange(201), np.arange(201), indexing="ij")
    mn = np.minimum(F, H)
    for rm in range(0, 41, 4):
        for rh in sorted(set(range(0, 41, 5)) | {rm, 40}):
            ready = (t[None, None, :] + rm < mn[..., None]) & (t[None, None, :] + rh < H[..., None])
            want = ready.sum(-1)                        # ready(t) is monotone in t, so the count is the prefix length
            got = np.vectorize(lambda f, h: landmark_counts(int(f), int(h), False, rm, rh))(F, H)
            assert np.array_equal(got, want), (rm, rh)
            assert np.array_equal(np.vectorize(lambda f, h: landmark_counts(int(f), int(h), True, rm, rh))(F, H), mn)
    for F_, H_, rm, rh in ((0, 0, 0, 0), (5, 3, 6, 40), (200, 200, 6, 40), (60, 60, 0, 0), (41, 41, 0, 40)):
        assert landmark_counts(F_, H_, False, rm, rh) == _brute(F_, H_, False, rm, rh)


@pytest.mark.parametrize("prm,lookahead", [(O.MAY, 55), (O.OBAMA1, 47)])
def test_portrait_counts_every_sample_count(prm, lookahead):
    p = _stage_params(prm)
    rm, rh = radii(p)
    prev = 0
    for n in range(0, 20001):
        c = ready_counts(n, False)
        got = portrait_counts(n, False, p)
        assert got == _brute(c.mouth, c.headpose, False, rm, rh)
        assert got >= prev
        prev = got
        end = ready_counts(n, True)
        assert portrait_counts(n, True, p) == min(end.mouth, end.headpose) >= got
    # frame t leaves once APC pair t + lookahead exists: pairs = t + lookahead + 1 ready
    for t in (0, 5, 100):
        pairs = t + lookahead + 1
        assert landmark_counts(max(0, pairs - 18), max(0, pairs - 15), False, rm, rh) == t + 1
        assert landmark_counts(max(0, pairs - 19), max(0, pairs - 16), False, rm, rh) == t


# ----------------------------------------------------------------------------------------------------------------------
# the live lip-fix truth
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", GOLDENS)
def test_live_truth_differs_only_on_outer_lips_of_crossed_frames(name):
    feat, head, ident, prm, pad = _golden(name)
    t, lt = O.truth(feat, head, ident, prm, pad), L.live_truth(feat, head, ident, prm, pad)
    outer = lt["outer"]
    for k in ("landmarks", "final_pts3d"):
        assert np.array_equal(t[k][~outer], lt[k][~outer]), k
    for k in ("shoulders", "pred_headpose"):
        assert np.array_equal(t[k], lt[k]), k
    flip = t["flip"]
    if flip.any():
        last = np.nonzero(flip)[0][-1]
        assert abs(lt["shift"][last] - lt["clip_shift"]) <= 1e-12 * abs(lt["clip_shift"])


def test_some_golden_has_running_and_clip_means_apart():
    apart = 0
    for name in GOLDENS:
        feat, head, ident, prm, pad = _golden(name)
        lt = L.live_truth(feat, head, ident, prm, pad)
        f = lt["flip"]
        apart += int(np.sum(np.abs(lt["shift"][f] - lt["clip_shift"]) > 1e-9))
    assert apart > 0


def _within(got, t, b):
    return max(float((np.abs(got[k] - t[k]) / b[k]).max()) if got[k].size else 0.0 for k in KEYS)


def _pushes(n_feat, n_head, size, seed=0):
    rng = np.random.default_rng(seed)
    out, f, h = [], 0, 0
    while f < n_feat or h < n_head:
        k = size if size else int(rng.integers(0, 12))
        out.append((k, k + (3 if h == 0 else 0)))
        f, h = f + k, h + k + (3 if h == 0 else 0)
    return out


@pytest.mark.parametrize("name", ["may_672", "obama1_672", "head_longer_300_340", "pad_200"])
def test_emulated_live_path_within_the_bound_and_defects_caught(name):
    feat, head, ident, prm, pad = _golden(name)
    lt = L.live_truth(feat, head, ident, prm, pad)
    b = O.error_bound(lt)
    for size in (1, 7, 0):
        got = L.emulate_live(feat, head, ident, prm, _pushes(*feat.shape[:1], head.shape[0], size, 1), pad)
        assert _within(got, lt, b) <= 1.0, size
    pushes = _pushes(feat.shape[0], head.shape[0], 7)
    for mutation in L.LIVE_MUTATIONS:
        got = L.emulate_live(feat, head, ident, prm, pushes, pad, mutation)
        assert _within(got, lt, b) > 1.0, mutation


# ----------------------------------------------------------------------------------------------------------------------
# LandmarkStream / PortraitStream bookkeeping with float64 stand-ins
# ----------------------------------------------------------------------------------------------------------------------
def _reflect(i, n):
    if n is None:                                           # the clip goes on: only the start folds back
        return i if i >= 0 else -1 - i
    return int(O.reflect_index(np.array([i]), n)[0])


class PostStandIn:
    """``lspl_run_stream``'s addressing in float64: every row it reads must be inside the window given.  Frame t's
    'landmarks' hold the gaussian-smoothed mouth columns, the smoothed head columns, the running lip shift and t % 37."""

    def __init__(self, rm, rh, widths=(16, 12)):
        self.rm, self.rh, self.widths = rm, rh, {75: widths[0], 6: widths[1]}
        self.wm, self.wh = (self._taps(r) for r in (rm, rh))

    @staticmethod
    def _taps(r):
        w = np.exp(-0.5 * (np.arange(-r, r + 1) / max(r / 4, 0.5)) ** 2)
        return w / w.sum()

    def stream(self, params, image_pad=None, return_intermediates=False):
        return LandmarkStream(self, params, image_pad, return_intermediates)

    def stream_state(self):
        return np.zeros(2)

    def device_rows(self, rows, width):
        return torch.as_tensor(np.asarray(rows, np.float64)).reshape(-1, self.widths[width])

    def _smooth(self, rows, row0, n_total, t, r, w):
        out = 0.0
        for k in range(-r, r + 1):
            i = _reflect(t + k, n_total) - row0
            assert 0 <= i < rows.shape[0], (t, k, row0, rows.shape[0])
            out = out + w[k + r] * rows[i]
        return out

    def run(self, feat, head):
        n = min(feat.shape[0], head.shape[0])
        st = self.stream_state()
        return self.run_stream(torch.as_tensor(feat), 0, torch.as_tensor(head), 0, 0, n, n, head.shape[0], None, st, None,
                               False)[0]

    def run_stream(self, feat, feat_row0, head, head_row0, frame0, n, nframe_total, n_head_total, native, state, ws,
                   return_intermediates):
        from livespeechportraits_b200.landmarks import LandmarkRows
        f, h = feat.numpy(), head.numpy()
        nm = None if nframe_total < 0 else nframe_total
        nh = None if n_head_total < 0 else n_head_total
        if frame0 == 0:
            state[:] = 0
        lm = np.zeros((n, 73, 2))
        for j in range(n):
            t = frame0 + j
            if nm is None:
                assert t + self.rm < min(feat_row0 + f.shape[0], head_row0 + h.shape[0])
            if nh is None:
                assert t + self.rh < head_row0 + h.shape[0]
            m = self._smooth(f, feat_row0, nm, t, self.rm, self.wm)
            p = self._smooth(h, head_row0, nh, t, self.rh, self.wh)
            if m[0] > 0:                                   # a 'crossed' frame
                state += (m[0], 1)
            v = np.concatenate([m, p, [state[0] / max(state[1], 1), t % 37]])
            lm[j].flat[:v.size] = v
        lm = torch.from_numpy(lm)
        return LandmarkRows(lm, lm[:, :18], frame0), ws


class NetStandIn:
    def draw_feature_maps(self, lm, sh, size, out=None):
        out[:] = (lm.reshape(lm.shape[0], 1, 1, -1).abs().sum(-1, keepdim=True) % 200).expand_as(out)
        return out

    def render_image(self, fm, cand, out=None):
        assert fm.shape[0] == 1 and out.shape[0] == 1                 # one frame per generator call
        out[:] = (fm.reshape(-1)[0] + cand.reshape(-1)[0]).to(out.dtype)
        return out


def _tracks(n_feat, n_head, seed):
    rng = np.random.default_rng(seed)
    return rng.normal(0, 1, (n_feat, 16)), rng.normal(0, 1, (n_head, 12))


@pytest.mark.parametrize("n_feat,n_head,rm,rh", [(300, 285, 6, 40), (60, 45, 4, 32), (30, 30, 0, 10), (5, 3, 6, 40),
                                                 (0, 0, 6, 40), (200, 230, 2, 8)])
def test_landmark_stream_chunks_give_the_whole_clip(n_feat, n_head, rm, rh):
    feat, head = _tracks(n_feat, n_head, n_feat)
    post = PostStandIn(rm, rh)
    whole = post.run(feat, head).landmarks.numpy()
    params = StageParams(rm / 4, "XYZ", [1, 1, 1], 1, 1, [rh / 4, rh / 4], 0.5)
    assert radii(params) == (rm, rh)
    for size in (1, 7, "random", max(n_feat, n_head, 1)):
        s = post.stream(params)
        outs, f, h = [], 0, 0
        rng = np.random.default_rng(3)
        while f < n_feat or h < n_head:
            k = int(rng.integers(0, 9)) if size == "random" else size
            df, dh = min(k, n_feat - f), min(k, n_head - h)
            r = s.push(feat[f:f + df], head[h:h + dh])
            f, h = f + df, h + dh
            assert r.frame0 == sum(o.shape[0] for o in outs) and s.frames == landmark_counts(f, h, False, rm, rh)
            assert s._feat_row0 == max(0, min(s.frames - rm, f)) and s._head_row0 == max(0, min(s.frames - rh, h))
            outs.append(r.landmarks.numpy())
        outs.append(s.finish().landmarks.numpy())
        got = np.concatenate(outs)
        assert got.shape == whole.shape and np.array_equal(got, whole), size
        with pytest.raises(RuntimeError):
            s.finish()


def test_portrait_stream_chunks_with_stand_ins():
    from test_stream_host import _sizes, _stand_ins
    mel, apc, mouth, head, opt, sd = _stand_ins()
    noise = np.random.default_rng(3).normal(0, 1, (4000, 12))
    params = StageParams(1.5, "XYZ", [2, 2, 2], 1, 0.5, [5, 10], 0.5)
    rm, rh = radii(params)
    audio = np.random.default_rng(5).uniform(-0.5, 0.5, 16000 * 2)
    cand = torch.zeros((1, 1, 8, 6), dtype=torch.float64)

    def session(sizes):
        a = AudioStream(mel, apc, mouth, head, pre_headpose=np.zeros(12), sigma_scale=0.3, noise=lambda i0, n: noise[i0:i0 + n])
        ps = PortraitStream(a, PostStandIn(rm, rh, (mouth.OUT, 12)), params, NetStandIn(), cand, size=(6, 8))
        outs, at = [], 0
        for k in sizes:
            r = ps.push(audio[at:at + k])
            at = min(at + k, audio.size)
            assert r.frame0 == sum(o.frames.shape[0] for o in outs) and ps.frames == portrait_counts(at, False, params)
            assert r.frames.shape[1:] == (8, 6, 3) and r.landmarks.shape[0] == r.frames.shape[0]
            outs.append(r)
        outs.append(ps.finish())
        assert ps.frames == portrait_counts(audio.size, True, params)
        return outs

    a = session(_sizes(audio.size, 1))
    b = session([267] * (audio.size // 267 + 1))
    for key in ("frames", "landmarks"):
        x = torch.cat([getattr(o, key) for o in a])
        y = torch.cat([getattr(o, key) for o in b])
        assert torch.equal(x, y), key
    lm = torch.cat([o.landmarks for o in a])
    assert lm.shape[0] > 0
    frames = torch.cat([o.frames for o in a])
    want = (lm.reshape(lm.shape[0], -1).abs().sum(-1) % 200).float()
    assert torch.equal(frames[:, 0, 0, 0], want.to(frames.dtype))


# ----------------------------------------------------------------------------------------------------------------------
# ABI checks on a host-only handle
# ----------------------------------------------------------------------------------------------------------------------
ENODEV, EINVAL = -2, -1


def test_run_stream_on_a_host_only_handle():
    lib = _lib.load()
    for name in ("lspl_stream_state_bytes", "lspl_stream_workspace_bytes", "lspl_run_stream"):
        assert getattr(lib, name).argtypes == _lib.ARGTYPES[name]
    h = C.c_void_p()
    assert lib.lspl_create(C.byref(h), -1) == 0
    P = 1 << 12
    try:
        sz = C.c_size_t()
        assert lib.lspl_stream_state_bytes(h, C.byref(sz)) == 0 and sz.value == 16
        assert lib.lspl_stream_workspace_bytes(h, 10, C.byref(sz)) == 0 and sz.value >= 10 * (54 * 8 + 6 * 4 + 8)
        assert lib.lspl_stream_workspace_bytes(h, -1, C.byref(sz)) == EINVAL
        prm = _lib.LsplParams(feat_sigma=1.5, rot_sigma=5, trans_sigma=10)        # rm 6, rh 40

        def run(f0=0, nf=100, h0=0, nh=100, frame0=10, n=5, nft=-1, nht=-1, state=P, params=prm, stride=12):
            return lib.lspl_run_stream(h, P, f0, nf, P, h0, nh, stride, frame0, n, nft, nht,
                                       C.byref(params) if params is not None else None, P, P, None, None, state, P,
                                       1 << 30, None)
        assert run() == ENODEV and b"no CPU path" in lib.lspl_last_error()
        assert run(state=None) == EINVAL and b"null state" in lib.lspl_last_error()
        assert run(params=None) == EINVAL and run(stride=5) == EINVAL
        assert run(frame0=-1) == EINVAL and run(n=-1) == EINVAL and run(nft=-2) == EINVAL
        assert run(frame0=(1 << 29) - 2, n=5) == EINVAL                        # frames end at or below 2^29
        # open clip: frame 14 needs mouth rows 8 .. 20 and head rows 0 .. 54
        assert run(nh=54) == EINVAL and b"head rows 0 .. 54" in lib.lspl_last_error()
        assert run(nh=55) == ENODEV
        assert run(f0=9, nh=55) == EINVAL and b"mouth rows 4 .. 20" in lib.lspl_last_error()
        assert run(f0=4, nf=17, nh=55) == ENODEV
        assert run(f0=4, nf=16, nh=55) == EINVAL
        assert run(nf=100, h0=1, nh=60) == EINVAL                              # head rows from 0
        # while nframe is open the mouth window must end before the head rows received
        assert run(nf=100, nh=20, n=5, frame0=10, nht=20) == EINVAL and b"not interior" in lib.lspl_last_error()
        # known totals: reflected windows stop at the totals; frames past them are refused
        assert run(nf=15, nh=15, frame0=10, n=5, nft=15, nht=15) == ENODEV
        assert run(nf=15, nh=15, frame0=10, n=6, nft=15, nht=15) == EINVAL and b"past the end" in lib.lspl_last_error()
        assert run(nf=14, nh=15, frame0=10, n=5, nft=15, nht=15) == EINVAL
        assert run(nft=16, nht=15, nf=16, nh=16) == EINVAL                     # nframe cannot exceed n_head
        assert run(f0=5, nf=3, h0=5, nh=3, frame0=0, n=0) == ENODEV            # nothing to emit
        assert run(nf=0, frame0=0, n=0, nh=0) == ENODEV
        assert run(frame0=0, n=1, nf=7, nh=41) == ENODEV                       # frame 0: rows from 0
    finally:
        assert lib.lspl_destroy(h) == 0
