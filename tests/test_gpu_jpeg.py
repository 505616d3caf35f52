"""The GPU JPEG encoder (include/lspj.h) against the numpy restatement (oracle/jpeg_oracle.py) and PIL: every slot's bytes
equal, at every quality, size, batch and channel count, for noise and for the generator's own frames and masks."""
import io
import threading
import types

import numpy as np
import pytest
import torch

from livespeechportraits_b200.jpeg import JpegEncoder
from oracle import jpeg_oracle as J

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0) if torch.cuda.is_available() else None

try:
    from PIL import Image
except ImportError:                                    # the oracle alone pins the bytes then
    Image = None


def _pil(img, q):
    if Image is None:
        return None
    b = io.BytesIO()
    Image.fromarray(img).save(b, "JPEG", quality=q)
    return b.getvalue()


def _images(n, h, w, grey, seed):
    rng = np.random.default_rng(seed)
    kinds = []
    for i in range(n):
        shape = (h, w) if grey else (h, w, 3)
        k = (seed + i) % 4
        if k == 0:
            a = rng.integers(0, 256, shape)
        elif k == 1:                                   # smooth gradient
            yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
            a = (xx * 255 // max(w - 1, 1) + yy * 3) % 256
            a = a if grey else np.stack([a, 255 - a, (a * 7) % 256], -1)
        elif k == 2:                                   # saturated 0/255
            a = rng.integers(0, 2, shape) * 255
        else:                                          # 8-px checkerboard
            yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
            a = ((yy // 8 + xx // 8) % 2) * 255
            a = a if grey else np.repeat(a[..., None], 3, -1)
        kinds.append(a.astype(np.uint8))
    return np.stack(kinds)


def _check(enc, imgs, q):
    batch = enc.encode(torch.from_numpy(imgs).to(DEV))
    files = batch.to_bytes()
    bound = enc.max_bytes(imgs.shape[1], imgs.shape[2], 1 if imgs.ndim == 3 else 3)
    for i, f in enumerate(files):
        want = J.encode(imgs[i], q)
        assert f == want, (i, q, imgs.shape, len(f), len(want))
        assert len(f) <= bound
        pil = _pil(imgs[i], q)
        assert pil is None or f == pil


@pytest.mark.parametrize("q", [1, 10, 50, 75, 90, 95, 100])
@pytest.mark.parametrize("grey", [False, True])
def test_every_quality_equals_the_oracle(q, grey):
    _check(JpegEncoder(DEV, quality=q), _images(7, 48, 64, grey, q), q)


@pytest.mark.parametrize("hw", [(16, 16), (256, 256), (512, 512), (256, 1024), (1024, 1024)])
@pytest.mark.parametrize("grey", [False, True])
def test_every_size_equals_the_oracle(hw, grey):
    _check(JpegEncoder(DEV, quality=75), _images(2, *hw, grey, hw[0] + hw[1]), 75)


@pytest.mark.parametrize("n", [1, 7, 32])
def test_batches_equal_the_oracle_frame_by_frame(n):
    imgs = _images(n, 64, 48, False, n)
    _check(JpegEncoder(DEV, quality=90), imgs, 90)


def test_generator_frames_and_masks_equal_the_oracle():
    from livespeechportraits_b200.generator import Feature2Face_G
    from oracle import f2f_oracle as O
    from oracle import raster_oracle as R
    net = Feature2Face_G(types.SimpleNamespace(isTrain=False, size="normal", n_downsample_G=8, ngf=64, fp16=0))
    net.load_state_dict(O.make_state_dict("normal", "B"), strict=True)
    net = net.to(DEV).eval()
    lm, sh = R.make_landmarks(3, (256, 256), seed=5, spill=0.1)
    maps = net.draw_feature_maps(torch.from_numpy(lm).to(DEV), torch.from_numpy(sh).to(DEV), (256, 256))
    _, cand = O.make_inputs(1, 256, 256)
    frames = torch.cat([net.render_image(maps[i:i + 1], cand.to(DEV)) for i in range(3)])
    masks = (maps[:, 0] * 255.0).to(torch.uint8)          # demo.py:270: np.uint8(map * 255)
    enc = JpegEncoder(DEV)
    _check(enc, frames.cpu().numpy(), 75)
    _check(enc, masks.cpu().numpy(), 75)


def test_encode_into_makes_no_host_synchronisation():
    enc = JpegEncoder(DEV)
    imgs = torch.from_numpy(_images(4, 256, 256, False, 1)).to(DEV)
    out = torch.empty((4, enc.max_bytes(256, 256)), dtype=torch.uint8, device=DEV)
    sizes = torch.empty(4, dtype=torch.int32, device=DEV)
    ws = torch.empty(enc.workspace_bytes(4, 256, 256, 3), dtype=torch.uint8, device=DEV)
    enc.encode_into(imgs, out, sizes, ws)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        enc.encode_into(imgs, out, sizes, ws)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    from livespeechportraits_b200.jpeg import JpegBatch
    assert JpegBatch(out, sizes).to_bytes() == [J.encode(a, 75) for a in imgs.cpu().numpy()]


def test_two_streams_equal_their_serial_results():
    """Two encoders, then one encoder whose two calls differ in batch size: every call has a workspace of its own."""
    a = torch.from_numpy(_images(8, 256, 256, False, 3)).to(DEV)
    b = torch.from_numpy(_images(8, 256, 256, True, 4)).to(DEV)
    shared = JpegEncoder(DEV, quality=75)
    for (ea, xa), (eb, xb) in (((JpegEncoder(DEV, quality=75), a), (JpegEncoder(DEV, quality=95), b)),
                               ((shared, a), (shared, b[:3]))):
        serial = (ea.encode(xa).to_bytes(), eb.encode(xb).to_bytes())
        sa, sb = torch.cuda.Stream(DEV), torch.cuda.Stream(DEV)
        torch.cuda.synchronize()
        with torch.cuda.stream(sa):
            ra = ea.encode(xa)
        with torch.cuda.stream(sb):
            rb = eb.encode(xb)
        torch.cuda.synchronize()
        assert (ra.to_bytes(), rb.to_bytes()) == serial


def test_encoders_on_two_threads_equal_their_serial_results():
    imgs = [torch.from_numpy(_images(4, 128, 128, False, s)).to(DEV) for s in (5, 6)]
    want = [[J.encode(x, 75) for x in i.cpu().numpy()] for i in imgs]
    got = [None, None]

    def run(k):
        with torch.cuda.stream(torch.cuda.Stream(DEV)):
            got[k] = JpegEncoder(DEV).encode(imgs[k]).to_bytes()

    ts = [threading.Thread(target=run, args=(k,)) for k in (0, 1)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert got == want
