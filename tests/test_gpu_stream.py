"""Streaming through demo.py stages 1-4 on the GPU (livespeechportraits_b200/stream.py and the stage ``.stream()`` objects):
every stream's concatenated output is compared with ``torch.equal`` against the whole-clip call on the same device."""
import functools
import os

import numpy as np
import pytest
import torch

from oracle import a2h_oracle as A
from oracle import lle_oracle as M
from oracle import mel_oracle as W
from oracle import rnn_oracle as R

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
MEL_DIR = os.path.join(os.path.dirname(__file__), "golden", "mel")


def _pieces(n, how, seed=0):
    """Piece sizes covering n: a fixed size, or seeded random sizes (zeros included)."""
    if how == "random":
        rng = np.random.default_rng(seed)
        out = []
        while sum(out) < n:
            out.append(int(rng.integers(0, max(2, n // 5))))
        return out
    return [how] * (n // how) + ([n % how] if n % how else [])


def _cat(parts, width):
    return torch.cat(parts) if parts else torch.empty((0, width), device=DEV)


# ----------------------------------------------------------------------------------------------------------------------
# mel
# ----------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _golden(name):
    return dict(np.load(os.path.join(MEL_DIR, name + ".npz")))


@pytest.mark.parametrize("how", [1, 37, 267, "random"])
@pytest.mark.parametrize("name", ["mel_00083_wav", "mel_synth_L200", "mel_synth_L199", "mel_synth_empty",
                                  "mel_synth_one_frame"])
def test_mel_stream_equals_logmel(name, how):
    from livespeechportraits_b200.audio import MelFrontEnd
    g = _golden(name)
    audio = g["audio"]
    if how == 1 and audio.shape[0] > 20000:
        audio = audio[:20000]                          # one-sample pushes: a prefix keeps the test short
    winlen, winstep = float(g["winlen"]), float(g["winstep"])
    front = MelFrontEnd(g["basis"], device=DEV)
    whole = front.logmel(audio, winlen=winlen, winstep=winstep)
    s = front.stream(winlen, winstep)
    parts, at = [], 0
    for k in _pieces(audio.shape[0], how, seed=len(name)):
        parts.append(s.push(audio[at:at + k]))
        at += k
    parts.append(s.finish())
    got = _cat(parts, whole.shape[1])
    assert got.shape == whole.shape and torch.equal(got, whole)


# ----------------------------------------------------------------------------------------------------------------------
# APC and Audio2Mouth
# ----------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _encoder(recipe, residual):
    from livespeechportraits_b200.recurrent import ApcEncoder
    return ApcEncoder(R.make_apc_state_dict(recipe, 0), device=DEV, residual=residual)


@pytest.mark.parametrize("how", [1, 7, "one"])
@pytest.mark.parametrize("cluster", [8, 16])
@pytest.mark.parametrize("T", [2, 37, 1374])
@pytest.mark.parametrize("recipe,residual", [("A", False), ("B", False), ("B", True)])
def test_apc_stream_equals_forward(recipe, residual, T, cluster, how):
    if how == 1 and T > 400:
        pytest.skip("one-row pushes on the long clip add minutes and no new case")
    enc = _encoder(recipe, residual)
    mel = torch.from_numpy(R.make_mel(T, seed=T)).to(DEV)
    whole = enc.forward(mel, cluster=cluster)
    s = enc.stream(cluster=cluster)
    parts, at = [], 0
    for k in _pieces(T, T if how == "one" else how):
        parts.append(s.push(mel[at:at + k]))
        at += k
    parts.append(s.finish())
    assert torch.equal(_cat(parts, 512), whole)


@functools.lru_cache(maxsize=None)
def _mouth(ff):
    from livespeechportraits_b200.recurrent import MouthGenerator
    opt = R.default_mouth_opt(frame_future=ff)
    return MouthGenerator(opt, R.make_mouth_state_dict(opt, "B", 0), device=DEV)


@pytest.mark.parametrize("how", [1, 5, "random", "one"])
@pytest.mark.parametrize("ff", [0, 18])
@pytest.mark.parametrize("n", [2, 36, 1374])
def test_mouth_stream_equals_generate(n, ff, how):
    gen = _mouth(ff)
    feats = torch.from_numpy(R.make_feats(n, seed=n)).to(DEV)
    whole = gen.generate(feats)
    s = gen.stream()
    parts, at = [], 0
    for k in _pieces(n, n if how == "one" else how, seed=n):
        parts.append(s.push(feats[at:at + k]))
        at = min(at + k, n)
        assert s.frames == (max(0, at // 2 - ff))            # a row comes out once its look-ahead pair is in
    parts.append(s.finish())
    got = _cat(parts, gen.out_dim)
    assert got.shape == whole.shape and torch.equal(got, whole)


# ----------------------------------------------------------------------------------------------------------------------
# head pose
# ----------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _headpose(ncenter=1):
    from livespeechportraits_b200.headpose import HeadposeGenerator
    opt = A.default_opt(A2H_GMM_ncenter=ncenter)
    return HeadposeGenerator(opt, A.make_state_dict(opt, "B", 1), device=DEV)


@pytest.mark.parametrize("how", [1, "random"])
@pytest.mark.parametrize("cluster", [1, 8])
@pytest.mark.parametrize("nframe", [1, 6, 300, 672])
def test_headpose_stream_equals_generate(nframe, cluster, how):
    if cluster == 1 and nframe == 672 and how == 1:
        pytest.skip("the single-CTA loop one frame at a time on the long clip adds minutes and no new case")
    gen = _headpose()
    ff = gen.cfg.frame_future
    n_audio = nframe + ff
    audio = torch.from_numpy(A.make_audio_feats(n_audio, A.default_opt(), 2)).to(DEV)
    noise = torch.from_numpy(A.reference_noise(nframe, 12, 1, seed=nframe))
    pre = torch.from_numpy(np.linspace(-0.1, 0.1, 12).astype(np.float32))
    whole, wparams = gen.generate(audio, pre, noise, 0.3, return_params=True, cluster=cluster)
    s = gen.stream(pre, 0.3, noise=lambda i0, n: noise[i0:i0 + n], return_params=True, cluster=cluster)
    preds, params, at = [], [], 0
    for k in _pieces(n_audio, how, seed=nframe):
        p, q = s.push(audio[at:at + k])
        at = min(at + k, n_audio)
        assert p.shape[0] == max(0, at - ff) - sum(x.shape[0] for x in preds)
        preds.append(p)
        params.append(q)
    p, q = s.finish()
    assert p.shape[0] == 0
    assert torch.equal(torch.cat(preds), whole) and torch.equal(torch.cat(params), wparams)


def test_headpose_stream_two_components_with_caller_uniform():
    gen = _headpose(2)
    nframe, ff = 40, gen.cfg.frame_future
    opt = A.default_opt(A2H_GMM_ncenter=2)
    audio = torch.from_numpy(A.make_audio_feats(nframe + ff, opt, 4)).to(DEV)
    noise = torch.from_numpy(A.reference_noise(nframe, 12, 1, seed=3))
    uniform = torch.rand(nframe, generator=torch.Generator().manual_seed(5))
    pre = np.zeros(12, np.float32)
    whole = gen.generate(audio, pre, noise, 0.3, uniform=uniform)
    with pytest.raises(ValueError, match="mixture component"):
        gen.stream(pre, 0.3)
    s = gen.stream(pre, 0.3, noise=lambda i0, n: (noise[i0:i0 + n], uniform[i0:i0 + n]))
    got = torch.cat([s.push(audio[i:i + 3]) for i in range(0, nframe + ff, 3)])
    assert torch.equal(got, whole)


# ----------------------------------------------------------------------------------------------------------------------
# the whole session
# ----------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _stages():
    from livespeechportraits_b200.audio import MelFrontEnd
    from livespeechportraits_b200.manifold import ManifoldProjector
    from livespeechportraits_b200.recurrent import ApcEncoder, MouthGenerator
    g = _golden("mel_00083_wav")
    mopt = R.default_mouth_opt()
    return (MelFrontEnd(g["basis"], device=DEV), ApcEncoder(R.make_apc_state_dict("B", 0), device=DEV),
            MouthGenerator(mopt, R.make_mouth_state_dict(mopt, "B", 0), device=DEV), _headpose(),
            ManifoldProjector(M.make_database(10_000, 512, seed=1), device=DEV))


def _whole_chain(audio, seed, projector=True):
    from livespeechportraits_b200.headpose import draw_reference_noise
    mel, apc, mouth, head, proj = _stages()
    feats = apc.forward(mel.logmel(audio))
    blend = proj.project_features(feats, 10, 1.0) if projector else feats
    torch.manual_seed(seed)
    nframe = blend.shape[0] // 2 - head.cfg.frame_future
    noise, _ = draw_reference_noise(nframe, 12, 1)
    return mouth.generate(blend), head.generate(blend.view(-1, 1024), np.zeros(12, np.float32), noise, 0.3)


def _stream_chain(audio, sizes, seed, projector=True, on_push=None):
    from livespeechportraits_b200.stream import AudioStream
    mel, apc, mouth, head, proj = _stages()
    torch.manual_seed(seed)
    s = AudioStream(mel, apc, mouth, head, projector=proj if projector else None, k=10, percent=1.0, sigma_scale=0.3)
    mouths, heads, at = [], [], 0
    for j, k in enumerate(sizes):
        r = s.push(audio[at:at + k])
        at += k
        assert r.mouth_frame0 == sum(x.shape[0] for x in mouths) and r.headpose_frame0 == sum(x.shape[0] for x in heads)
        mouths.append(r.mouth)
        heads.append(r.headpose)
        if on_push:
            on_push(j, mouths, heads)
    r = s.finish()
    return torch.cat([x.to(DEV) for x in mouths + [r.mouth]]), torch.cat([x.to(DEV) for x in heads + [r.headpose]])


@pytest.mark.parametrize("how", [267, "random"])
def test_session_equals_the_whole_clip_chain(how):
    audio = _golden("mel_00083_wav")["audio"]
    wm, wh = _whole_chain(audio, seed=7)
    sm, sh = _stream_chain(audio, _pieces(audio.shape[0], how, seed=11), seed=7)
    assert sm.shape == wm.shape and sh.shape == wh.shape == (687 - 15, 12)
    assert torch.equal(sm, wm) and torch.equal(sh, wh)


def test_session_memory_is_bounded_over_ten_minutes():
    audio = W.make_audio(16000 * 600, seed=4)
    wm, wh = _whole_chain(audio, seed=2, projector=False)
    wm, wh = wm.cpu(), wh.cpu()
    torch.cuda.synchronize()
    seen = {}

    def on_push(j, mouths, heads):
        mouths[-1], heads[-1] = mouths[-1].cpu(), heads[-1].cpu()       # the caller keeps its rows on the host
        seen[j] = torch.cuda.memory_allocated(DEV)
    sm, sh = _stream_chain(audio, [16000] * 600, seed=2, projector=False, on_push=on_push)
    changes = [(j, seen[j] - seen[j - 1]) for j in range(1, 600) if seen[j] != seen[j - 1]]
    assert seen[9] == seen[599], (seen[9], seen[599], changes[:20])
    assert torch.equal(sm.cpu(), wm) and torch.equal(sh.cpu(), wh)
