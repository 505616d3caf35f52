"""librosa.load's resampling on the GPU (``audio.Resampler``, ``ResampleStream``; include/lspa.h ``lspa_resample_at``):
whole clips ``torch.equal`` to the oracle restatement (oracle/resample_oracle.py) for every input rate, both tables,
both sample formats and one or two channels; a 40-minute clip at the register's binade boundaries; streams over several
chunkings against the whole clip; and the live path (``AudioStream``, ``PortraitStream``) fed 48 kHz PCM16 stereo
against the same streams fed the whole-clip 16 kHz samples, with no synchronising push and bounded device memory."""
import functools
import types

import numpy as np
import pytest
import torch

from oracle import resample_oracle as R
from test_gpu_stream import _pieces, _stages

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
RATES = [8000, 11025, 22050, 24000, 32000, 44100, 48000, 96000]


@functools.lru_cache(maxsize=None)
def _resampler(orig_sr, channels, name):
    from livespeechportraits_b200.audio import Resampler
    return Resampler(orig_sr, channels, name, device=DEV)


def _frames(n, channels, dtype, seed):
    rng = np.random.default_rng(seed)
    shape = (n,) if channels == 1 else (n, channels)
    if dtype == np.int16:
        return rng.integers(-32768, 32768, size=shape, dtype=np.int16)
    return (0.3 * rng.standard_normal(shape)).astype(np.float32)


def _check(rs, frames, orig_sr, name, outputs=None):
    got = rs.resample(frames)
    want_len = int(np.ceil(frames.shape[0] * 16000.0 / orig_sr))
    assert got.shape == (want_len,) and got.dtype == torch.float32 and got.device == DEV
    want = torch.from_numpy(R.resample(frames, orig_sr, name, outputs=outputs)).to(DEV)
    sel = got if outputs is None else got[torch.from_numpy(outputs).to(DEV)]
    assert torch.equal(sel, want), (orig_sr, name, frames.shape, frames.dtype, int((sel != want).sum()))


def _chosen(n_out, seed):
    """Output indices: both ends and a seeded spread in between."""
    rng = np.random.default_rng(seed)
    return np.unique(np.concatenate([np.arange(min(600, n_out)), np.arange(max(0, n_out - 600), n_out),
                                     rng.integers(0, n_out, size=1500)]))


@pytest.mark.parametrize("fmt,channels", [(np.float32, 1), (np.float32, 2), (np.int16, 1), (np.int16, 2)])
@pytest.mark.parametrize("name", ["kaiser_best", "kaiser_fast"])
@pytest.mark.parametrize("orig_sr", RATES)
def test_whole_clip_equals_the_restatement(orig_sr, name, fmt, channels):
    rs = _resampler(orig_sr, channels, name)
    ratio = 16000.0 / orig_sr
    shortest = next(n for n in range(1, 100) if int(n * ratio) >= 1)
    with pytest.raises(ValueError, match="too small"):
        rs.resample(_frames(shortest - 1, channels, fmt, 0))
    for n in (shortest, shortest + 1, 1001, 4099, orig_sr // 3 + 7):
        _check(rs, _frames(n, channels, fmt, n), orig_sr, name)
    for seconds in (183296 / 16000, 60):                 # the 00083.wav duration, and a minute
        n = int(seconds * orig_sr) | 1
        _check(rs, _frames(n, channels, fmt, n), orig_sr, name, _chosen(int(np.ceil(n * ratio)), n))


def test_whole_clip_from_torch_on_the_device():
    frames = _frames(48000 * 3 + 5, 2, np.int16, 3)
    rs = _resampler(48000, 2, "kaiser_best")
    assert torch.equal(rs.resample(torch.from_numpy(frames).to(DEV)), rs.resample(frames))


def test_sixteen_khz_is_the_mono_mix():
    from livespeechportraits_b200.audio import Resampler
    frames = _frames(16001, 2, np.int16, 4)
    got = Resampler(16000, 2, device=DEV).resample(frames)
    assert torch.equal(got.cpu(), torch.from_numpy(np.mean(R.decode(frames).T, axis=0)))


def test_forty_minutes_at_the_register_binades():
    """The register crosses 2^k at output ~ 2^k / 2.76; the outputs around each crossing from 2^11 on."""
    orig_sr, name = 44100, "kaiser_best"
    n = 40 * 60 * orig_sr + 1
    frames = _frames(n, 1, np.int16, 40)
    rs = _resampler(orig_sr, 1, name)
    got = rs.resample(frames)
    ratio = 16000.0 / orig_sr
    n_out = int(n * ratio)
    cross = [int(2 ** k * ratio) for k in range(11, 40) if 2 ** k * ratio < n_out - 64]
    assert len(cross) >= 15
    sel = np.unique(np.concatenate([np.arange(c - 40, c + 40) for c in cross] + [np.arange(n_out - 300, n_out + 1)]))
    want = torch.from_numpy(R.resample(frames, orig_sr, name, outputs=sel)).to(DEV)
    assert torch.equal(got[torch.from_numpy(sel).to(DEV)], want)


# ----------------------------------------------------------------------------------------------------------------------
# streaming
# ----------------------------------------------------------------------------------------------------------------------
def _stream(rs, frames, sizes):
    s = rs.stream()
    parts, at = [], 0
    for k in sizes:
        parts.append(s.push(frames[at:at + k]))
        at += k
    parts.append(s.finish())
    assert s.samples == sum(p.shape[0] for p in parts)
    return torch.cat(parts)


@pytest.mark.parametrize("orig_sr,channels,fmt,name", [(48000, 2, np.int16, "kaiser_best"),
                                                       (44100, 1, np.float32, "kaiser_best"),
                                                       (8000, 1, np.int16, "kaiser_fast"),
                                                       (22050, 2, np.float32, "kaiser_fast"),
                                                       (96000, 1, np.int16, "kaiser_best")])
@pytest.mark.parametrize("how", [1, "10ms", "random", "one"])
def test_stream_equals_the_whole_clip(orig_sr, channels, fmt, name, how):
    rs = _resampler(orig_sr, channels, name)
    n = 3001 if how == 1 else orig_sr * 3 + 333
    frames = _frames(n, channels, fmt, n + orig_sr)
    sizes = _pieces(n, {"10ms": orig_sr // 100, "one": n}.get(how, how), seed=orig_sr)
    got = _stream(rs, frames, sizes)
    whole = rs.resample(frames)
    assert got.shape == whole.shape and torch.equal(got, whole)


def test_stream_refuses_what_resampy_refuses():
    s = _resampler(48000, 1, "kaiser_best").stream()
    assert s.push(np.zeros(2, np.float32)).shape == (0,)
    with pytest.raises(ValueError, match="too small"):
        s.finish()


# ----------------------------------------------------------------------------------------------------------------------
# the live path: 48 kHz PCM16 stereo in 10 ms pushes
# ----------------------------------------------------------------------------------------------------------------------
SIZE = 512


@functools.lru_cache(maxsize=1)
def _large():
    from livespeechportraits_b200.generator import Feature2Face_G
    from oracle import f2f_oracle as F
    net = Feature2Face_G(types.SimpleNamespace(isTrain=False, size="large", n_downsample_G=8, ngf=64, fp16=0),
                         precision="parity")
    net.load_state_dict(F.make_state_dict("large", "B"))
    _, cand = F.make_inputs(1, SIZE, SIZE, seed=6)
    return net.to(DEV).eval(), cand[:1].to(DEV)


def _portrait(feed, resampler, size=SIZE, net=None, projector=True, on_push=None):
    from livespeechportraits_b200.landmarks import Identity, LandmarkPostprocessor
    from livespeechportraits_b200.stream import AudioStream, PortraitStream
    from oracle import landmark_oracle as O
    from test_gpu_landmarks import _params
    mel, apc, mouth, head, proj = _stages()
    net, cand = net or _large()
    torch.manual_seed(5)
    a = AudioStream(mel, apc, mouth, head, projector=proj if projector else None, k=10, percent=1.0, sigma_scale=0.3,
                    resampler=resampler)
    ps = PortraitStream(a, LandmarkPostprocessor(Identity(**O.make_identity(0, 37)), device=DEV), _params(O.MAY), net,
                        cand, size=(size, size))
    outs = []
    for j, piece in enumerate(feed):
        outs.append(ps.push(piece))
        if on_push:
            on_push(j, outs)
    outs.append(ps.finish())
    return outs


def test_live_path_fed_48k_pcm16_stereo_equals_the_16k_feed():
    from livespeechportraits_b200.audio import Resampler
    rs = Resampler(48000, 2, device=DEV)
    frames = _frames(48000 * 3 + 123, 2, np.int16, 9)
    pcm = [frames[i:i + 480] for i in range(0, frames.shape[0], 480)]
    audio16 = rs.resample(frames)
    s16 = [audio16[i:i + 160] for i in range(0, audio16.shape[0], 160)]
    native, ref = _portrait(pcm, rs), _portrait(s16, None)
    for key in ("mouth", "headpose", "apc", "features"):
        a = torch.cat([getattr(o.rows, key) for o in native])
        b = torch.cat([getattr(o.rows, key) for o in ref])
        assert a.shape == b.shape and torch.equal(a, b), key
    for key in ("frames", "landmarks", "shoulders"):
        a, b = torch.cat([getattr(o, key) for o in native]), torch.cat([getattr(o, key) for o in ref])
        assert a.shape == b.shape and torch.equal(a, b), key
    assert torch.cat([o.frames for o in native]).shape[1:] == (SIZE, SIZE, 3) and len(native) > 300


def test_live_push_makes_no_synchronising_call():
    from livespeechportraits_b200.audio import Resampler
    from livespeechportraits_b200.landmarks import Identity, LandmarkPostprocessor
    from livespeechportraits_b200.stream import AudioStream, PortraitStream
    from oracle import landmark_oracle as O
    from test_gpu_landmarks import _params
    from test_gpu_portrait_stream import _net
    frames = _frames(48000 * 2, 2, np.int16, 10)
    mel, apc, mouth, head, proj = _stages()
    net, cand = _net()
    torch.manual_seed(0)
    a = AudioStream(mel, apc, mouth, head, projector=proj, k=10, percent=1.0, sigma_scale=0.3,
                    resampler=Resampler(48000, 2, device=DEV))
    ps = PortraitStream(a, LandmarkPostprocessor(Identity(**O.make_identity(0, 37)), device=DEV), _params(O.MAY), net,
                        cand, size=(256, 256))
    at = 0
    while ps.frames < 3:
        ps.push(frames[at:at + 800])
        at += 800
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        r = ps.push(frames[at:at + 800])
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert r.frames.shape[0] == 1


def test_live_memory_is_bounded_over_two_minutes():
    from livespeechportraits_b200.audio import Resampler
    from test_gpu_portrait_stream import _net
    frames = _frames(48000 * 120, 2, np.int16, 11)
    seen = {}

    def on_push(j, outs):
        outs[-1] = None                                     # the caller keeps nothing on the device
        seen[j] = torch.cuda.memory_allocated(DEV)
    _portrait([frames[i:i + 48000] for i in range(0, frames.shape[0], 48000)], Resampler(48000, 2, device=DEV),
              size=256, net=_net(), projector=False, on_push=on_push)
    assert seen[9] == seen[119], (seen[9], seen[119])
