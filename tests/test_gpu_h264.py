"""The GPU H.264 encoder (include/lspv.h) against the numpy restatement (oracle/h264_oracle.py): every access unit's bytes
and every reconstructed frame equal, over the case matrix, on the generator's frames and masks and on the goldens
(whose planes libavcodec decoded); pushes equal the whole clip, runs repeat, sizes stay under lspv_max_bytes."""
import json
import os
import types

import numpy as np
import pytest
import torch

from h264_cases import CASES, case_id, clip
from livespeechportraits_b200.h264 import H264Encoder
from oracle import h264_oracle as H

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0) if torch.cuda.is_available() else None
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "h264")


def _planes(state: torch.Tensor, h: int, w: int):
    s = state.cpu().numpy()[256:]
    return s[:h * w].reshape(h, w), s[h * w:h * w * 5 // 4].reshape(h // 2, w // 2), \
        s[h * w * 5 // 4:h * w * 3 // 2].reshape(h // 2, w // 2)


def _encode_frames(enc: H264Encoder, frames: np.ndarray):
    """Frame by frame through a stream: (access units, IDR flags, reconstruction after each frame)."""
    st = enc.stream()
    aus, idrs, recs = [], [], []
    h, w = frames.shape[1:3]
    for f in frames:
        b = st.push(torch.from_numpy(f[None]).to(DEV))
        aus += b.to_bytes()
        idrs += [bool(x) for x in b.is_idr.cpu().tolist()]
        recs.append(_planes(st.state, h, w))
    return aus, idrs, recs, st


@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_bytes_and_reconstruction_equal_the_oracle(case):
    kind, h, w, qp, gop, search, n = case
    frames = clip(kind, n, h, w, seed=h + w + qp)
    enc = H264Encoder(DEV, qp=qp, gop=gop, search=search)
    aus, idrs, recs, st = _encode_frames(enc, frames)
    want, widr, wrec, _ = H.encode(frames, qp=qp, gop=gop, search=search)
    bound = enc.max_bytes(h, w)
    assert H.max_bytes(h, w) == bound
    for i in range(n):
        assert aus[i] == want[i], (i, len(aus[i]), len(want[i]))
        assert idrs[i] == widr[i] == (i % gop == 0)
        for k in range(3):
            assert np.array_equal(recs[i][k], wrec[i][k]), (i, k)
        assert len(aus[i]) <= bound
    assert int(st.state[:8].cpu().view(torch.int64)) == n                      # the state's next-frame index


def _generator_frames(n, size):
    from livespeechportraits_b200.generator import Feature2Face_G
    from oracle import f2f_oracle as O
    from oracle import raster_oracle as R
    net = Feature2Face_G(types.SimpleNamespace(isTrain=False, size="large", n_downsample_G=8, ngf=64, fp16=0))
    net.load_state_dict(O.make_state_dict("large", "B"), strict=True)
    net = net.to(DEV).eval()
    lm, sh = R.make_landmarks(n, (size, size), seed=5, spill=0.1)
    maps = net.draw_feature_maps(torch.from_numpy(lm).to(DEV), torch.from_numpy(sh).to(DEV), (size, size))
    _, cand = O.make_inputs(1, size, size)
    frames = torch.cat([net.render_image(maps[i:i + 1], cand.to(DEV)) for i in range(n)])
    return frames, (maps[:, 0] * 255.0).to(torch.uint8)


def test_generator_frames_and_masks_equal_the_oracle():
    frames, masks = _generator_frames(3, 512)
    for imgs in (frames, masks):
        enc = H264Encoder(DEV, qp=26, gop=60)
        got = enc.encode(imgs).to_bytes()
        want, _, _, _ = H.encode(imgs.cpu().numpy(), qp=26, gop=60)
        assert got == want, [(len(a), len(b)) for a, b in zip(got, want)]


def test_goldens_decode_as_libavcodec_did():
    cases = json.load(open(os.path.join(GOLDEN, "cases.json")))
    for c in cases:
        frames = clip(c["kind"], c["frames"], c["height"], c["width"], seed=c["seed"])
        enc = H264Encoder(DEV, qp=c["qp"], gop=c["gop"], search=c["search"])
        aus, _, recs, _ = _encode_frames(enc, frames)
        stream = open(os.path.join(GOLDEN, c["name"] + ".h264"), "rb").read()
        assert b"".join(aus) == stream, c["name"]
        planes = np.load(os.path.join(GOLDEN, c["name"] + ".npz"))
        for i, r in enumerate(recs):
            for k, p in enumerate("yuv"):
                assert np.array_equal(r[k], planes[f"{p}{i}"]), (c["name"], i, p)


@pytest.mark.parametrize("push", [1, 7, 32])
def test_pushes_equal_the_whole_clip(push):
    frames = clip("smooth", 70, 64, 96, seed=2)
    enc = H264Encoder(DEV, qp=30, gop=60, search=8)
    imgs = torch.from_numpy(frames).to(DEV)
    whole = enc.encode(imgs)
    st = enc.stream()
    parts = []
    for at in range(0, 70, push):
        parts += st.push(imgs[at:at + push]).to_bytes()
    parts += st.finish().to_bytes()
    assert parts == whole.to_bytes()
    assert whole.is_idr.cpu().tolist() == [1 if i % 60 == 0 else 0 for i in range(70)]


def test_two_streams_of_one_encoder_on_two_cuda_streams_equal_their_serial_results():
    """Each H264Stream owns its workspace, so two streams of one encoder, pushing clips of different sizes on two CUDA
    streams with nothing ordering one's pushes against the other's, give the bytes and reconstruction of a serial run."""
    enc = H264Encoder(DEV, qp=26, gop=4, search=8)
    clips = [torch.from_numpy(clip("noise", 6, 256, 256, seed=1)).to(DEV),
             torch.from_numpy(clip("translate", 6, 128, 192, seed=2)).to(DEV)]
    want = []
    for x in clips:
        st = enc.stream()
        want.append((st.push(x).to_bytes(), st.state.cpu()))
    cuda_streams, streams = [torch.cuda.Stream(DEV) for _ in clips], [enc.stream() for _ in clips]
    got = [[], []]
    torch.cuda.synchronize()
    for at in range(0, 6, 2):
        for k in (0, 1):
            with torch.cuda.stream(cuda_streams[k]):
                got[k].append(streams[k].push(clips[k][at:at + 2]))
    torch.cuda.synchronize()
    for k in (0, 1):
        assert [au for b in got[k] for au in b.to_bytes()] == want[k][0], k
        assert torch.equal(streams[k].state.cpu(), want[k][1]), k


def test_two_runs_give_identical_bytes_under_the_bound():
    frames, _ = _generator_frames(4, 512)
    frames = torch.cat([frames, torch.from_numpy(clip("noise", 2, 512, 512)).to(DEV)])
    enc = H264Encoder(DEV, qp=0, gop=3)
    a, b = enc.encode(frames), enc.encode(frames)
    assert a.to_bytes() == b.to_bytes()
    assert int(a.sizes.max()) <= enc.max_bytes(512, 512)


def test_encode_makes_no_host_synchronisation():
    enc = H264Encoder(DEV, qp=26, gop=4)
    imgs = torch.from_numpy(clip("smooth", 6, 128, 128)).to(DEV)
    st = enc.stream()
    st.push(imgs[:1])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        b = st.push(imgs[1:])
    finally:
        torch.cuda.set_sync_debug_mode("default")
    want, _, _, _ = H.encode(imgs.cpu().numpy(), qp=26, gop=4)
    assert b.to_bytes() == want[1:]
