"""Live stage 5 and live portraits on the GPU: ``LandmarkStream`` (include/lspl.h ``lspl_run_stream``) against
``LandmarkPostprocessor.run`` on the whole tracks (``torch.equal`` everywhere but the outer lips of crossed frames, which
follow the running-mean rule within the bound of ``live_truth``), and ``stream.PortraitStream`` against the whole-clip
chain, with no synchronising call in a push and bounded device memory."""
import functools
import types

import numpy as np
import pytest
import torch

import live_landmark_oracle as L
from oracle import landmark_oracle as O
from test_gpu_landmarks import GOLDENS, KEYS, _golden, _params
from test_gpu_stream import _pieces, _stages
from test_gpu_stream import _golden as _mel_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _post_of(ident):
    from livespeechportraits_b200.landmarks import Identity, LandmarkPostprocessor
    return LandmarkPostprocessor(Identity(**ident), device=DEV)


def _stream(post, feat, head, prm, pad, how, seed=0):
    """feat and head pushed together in pieces (sizes `how`), then finished: the concatenated outputs."""
    s = post.stream(_params(prm), image_pad=pad, return_intermediates=True)
    n = max(feat.shape[0], head.shape[0])
    parts, at = [], 0
    for k in _pieces(n, how, seed) if n else []:
        r = s.push(feat[at:at + k], head[at:at + k])
        assert r.frame0 == sum(p[0].shape[0] for p in parts)
        parts.append(tuple(r[i] for i in (0, 1, 3, 4)))
        at += k
    r = s.finish()
    parts.append(tuple(r[i] for i in (0, 1, 3, 4)))
    return [torch.cat([p[i] for p in parts]) for i in range(4)]


def _check_live(post, feat, head, ident, prm, pad, label):
    f, h = torch.from_numpy(feat).to(DEV), torch.from_numpy(head).to(DEV)
    whole = post.run(f, h, _params(prm), image_pad=pad, return_intermediates=True)
    lt = L.live_truth(feat, head, ident, prm, pad)
    b = O.error_bound(lt)
    outer = torch.from_numpy(lt["outer"]).to(DEV)
    first = None
    for how in (1, 7, "random", max(feat.shape[0], head.shape[0], 1)):
        got = _stream(post, f, h, prm, pad, how, seed=len(label))
        for k, g, w in zip(KEYS, got, whole):
            assert g.shape == w.shape, (label, how, k)
            if k in ("landmarks", "final_pts3d"):
                assert torch.equal(g[~outer], w[~outer]), (label, how, k)
            else:
                assert torch.equal(g, w), (label, how, k)
        for k, g in zip(KEYS, got):
            ratio = float((np.abs(g.cpu().numpy() - lt[k]) / b[k]).max()) if g.numel() else 0.0
            assert ratio <= 1.0, (label, how, k, ratio)
        if first is None:
            first = got
        assert all(torch.equal(a, c) for a, c in zip(first, got)), (label, how)
    return int(lt["flip"].sum())


@pytest.mark.parametrize("name", GOLDENS)
def test_landmark_stream_goldens(name):
    feat, head, ident, prm, pad, _ = _golden(name)
    _check_live(_post_of(ident), feat, head, ident, prm, pad, name)


@pytest.mark.parametrize("n_feat,n_head", [(3, 3), (33, 33), (65, 64), (64, 65), (100, 1), (1, 100), (500, 97)])
def test_landmark_stream_other_lengths(n_feat, n_head):
    ident = O.make_identity(0, 37)
    feat, head = O.make_tracks(n_feat, n_head, n_feat + n_head)
    _check_live(_post_of(ident), feat, head, ident, O.MAY, None, f"{n_feat}x{n_head}")


@pytest.mark.parametrize("cross,prm", [(0.3, O.MAY), (0.5, O.OBAMA1), (0.3, dict(O.MAY, Feat_smooth_sigma=0))])
def test_landmark_stream_crossing_heavy(cross, prm):
    ident = O.make_identity(1, 37)
    feat, head = O.make_tracks(400, 415, 9, cross=cross)
    crossed = _check_live(_post_of(ident), feat, head, ident, prm, (3, 5, 7, 11), f"cross {cross}")
    assert crossed > 100


def test_landmark_stream_empty_clips():
    ident = O.make_identity(0, 37)
    post = _post_of(ident)
    for nf, nh in ((0, 10), (10, 0), (0, 0)):
        got = _stream(post, torch.zeros((nf, 75), device=DEV), torch.zeros((nh, 12), device=DEV), O.MAY, None, 3)
        assert got[0].shape == (0, 73, 2) and got[1].shape == (0, 18, 2)


# ----------------------------------------------------------------------------------------------------------------------
# PortraitStream: audio in, frames out
# ----------------------------------------------------------------------------------------------------------------------
SIZE = 256


@functools.lru_cache(maxsize=1)
def _net():
    from livespeechportraits_b200.generator import Feature2Face_G
    from oracle import f2f_oracle as F
    net = Feature2Face_G(types.SimpleNamespace(isTrain=False, size="normal", n_downsample_G=8, ngf=64, fp16=0),
                         precision="parity")
    net.load_state_dict(F.make_state_dict("normal", "B"))
    _, cand = F.make_inputs(1, SIZE, SIZE, seed=6)
    return net.to(DEV).eval(), cand[:1].to(DEV)


def _render_each(net, cand, lm, sh):
    maps = net.draw_feature_maps(lm, sh, (SIZE, SIZE))
    return torch.cat([net.render_image(maps[i:i + 1], cand) for i in range(lm.shape[0])]) if lm.shape[0] else \
        torch.empty((0, SIZE, SIZE, 3), dtype=torch.uint8, device=DEV)


def _portrait(audio, sizes, seed, projector=True, on_push=None):
    from livespeechportraits_b200.stream import AudioStream, PortraitStream
    mel, apc, mouth, head, proj = _stages()
    net, cand = _net()
    ident = O.make_identity(0, 37)
    torch.manual_seed(seed)
    a = AudioStream(mel, apc, mouth, head, projector=proj if projector else None, k=10, percent=1.0, sigma_scale=0.3)
    ps = PortraitStream(a, _post_of(ident), _params(O.MAY), net, cand, size=(SIZE, SIZE))
    outs, at = [], 0
    for j, k in enumerate(sizes):
        r = ps.push(audio[at:at + k])
        at += k
        assert r.frame0 == sum(o[0].shape[0] for o in outs)
        outs.append([r.frames, r.landmarks, r.shoulders])
        if on_push:
            on_push(j, outs)
    r = ps.finish()
    outs.append([r.frames, r.landmarks, r.shoulders])
    return [torch.cat([o[i].to(DEV) for o in outs]) for i in range(3)], ident


@pytest.mark.parametrize("how", [267, "random"])
def test_portrait_stream_equals_the_whole_clip_chain(how):
    from test_gpu_stream import _whole_chain
    audio = _mel_golden("mel_00083_wav")["audio"]
    wm, wh = _whole_chain(audio, seed=7)
    (frames, lm, sh), ident = _portrait(audio, _pieces(audio.shape[0], how, seed=11), seed=7)
    post = _post_of(ident)
    wlm, wsh, wpts, _ = post.run(wm, wh, _params(O.MAY), return_intermediates=True)
    net, cand = _net()
    wframes = _render_each(net, cand, wlm, wsh)
    assert lm.shape == wlm.shape and frames.shape == (lm.shape[0], SIZE, SIZE, 3)
    lt = L.live_truth(wm.cpu().numpy(), wh.cpu().numpy().astype(np.float64), ident, O.MAY)
    outer = torch.from_numpy(lt["outer"]).to(DEV)
    assert torch.equal(lm[~outer], wlm[~outer]) and torch.equal(sh, wsh)
    same = (lm == wlm).flatten(1).all(1)
    assert torch.equal(frames[same], wframes[same])
    assert torch.equal(frames, _render_each(net, cand, lm, sh))
    print(f"{how}: {lm.shape[0]} frames, {int(same.sum())} with landmarks bit-equal to the whole clip's")


def test_portrait_push_makes_no_synchronising_call():
    from livespeechportraits_b200.stream import AudioStream, PortraitStream
    audio = _mel_golden("mel_00083_wav")["audio"]
    mel, apc, mouth, head, proj = _stages()
    net, cand = _net()
    torch.manual_seed(0)
    a = AudioStream(mel, apc, mouth, head, projector=proj, k=10, percent=1.0, sigma_scale=0.3)
    ps = PortraitStream(a, _post_of(O.make_identity(0, 37)), _params(O.MAY), net, cand, size=(SIZE, SIZE))
    at = 0
    while ps.frames < 3:
        ps.push(audio[at:at + 267])
        at += 267
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        r = ps.push(audio[at:at + 267])
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert r.frames.shape[0] == 1


def test_portrait_stream_memory_is_bounded_over_two_minutes():
    from oracle import mel_oracle as W
    audio = W.make_audio(16000 * 120, seed=5)
    seen = {}

    def on_push(j, outs):
        outs[-1] = [x.cpu() for x in outs[-1]]              # the caller keeps its frames on the host
        seen[j] = torch.cuda.memory_allocated(DEV)
    (frames, lm, _), _ = _portrait(audio, [16000] * 120, seed=2, projector=False, on_push=on_push)
    assert frames.shape[0] == lm.shape[0] > 7000
    assert seen[9] == seen[119], (seen[9], seen[119])
