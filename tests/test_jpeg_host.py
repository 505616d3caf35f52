"""The JPEG restatement (oracle/jpeg_oracle.py) against PIL and cv2.imencode (two libjpeg-turbo builds), the bound
lspj_max_bytes, and the host-only checks of include/lspj.h."""
import ctypes as C
import io
import json
import os
import re

import numpy as np
import pytest

from livespeechportraits_b200 import _lib
from oracle import jpeg_oracle as J

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "jpeg")

try:
    from PIL import Image
except ImportError:
    Image = None
try:
    import cv2
except ImportError:
    cv2 = None


def _pil(img, q):
    b = io.BytesIO()
    Image.fromarray(img).save(b, "JPEG", quality=q)
    return b.getvalue()


def _cv2(img, q):
    return cv2.imencode(".jpg", img[..., ::-1] if img.ndim == 3 else img, [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes()


def _both(img, q):
    got = J.encode(img, q)
    if Image is None and cv2 is None:
        pytest.skip("neither PIL nor cv2 is importable")
    if Image is not None:
        assert got == _pil(img, q)
    if cv2 is not None:
        assert got == _cv2(img, q)


def _pattern(kind, h, w, grey, seed=0):
    rng = np.random.default_rng(seed)
    shape = (h, w) if grey else (h, w, 3)
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    if kind == "noise":
        a = rng.integers(0, 256, shape)
    elif kind == "gradient":
        a = (xx * 255 // max(w - 1, 1) + yy) % 256
        a = a if grey else np.stack([a, (yy * 255 // max(h - 1, 1)) % 256, 255 - a], -1)
    elif kind == "saturated":
        a = rng.integers(0, 2, shape) * 255
    else:
        cell = 1 if kind == "checker1" else 8
        a = ((yy // cell + xx // cell) % 2) * 255
        a = a if grey else np.stack([a, 255 - a, a], -1)
    return a.astype(np.uint8)


@pytest.mark.parametrize("grey", [False, True])
def test_every_quality_equals_pil_and_cv2(grey):
    img = _pattern("noise", 32, 48, grey, seed=4)
    for q in range(1, 101):
        _both(img, q)


@pytest.mark.parametrize("hw", [(16, 16), (48, 32), (256, 512), (512, 512)])
@pytest.mark.parametrize("kind", ["noise", "gradient", "saturated", "checker1", "checker8"])
@pytest.mark.parametrize("grey", [False, True])
def test_sizes_and_patterns_equal_pil_and_cv2(hw, kind, grey):
    if hw[0] * hw[1] > 48 * 32 and kind in ("checker1", "saturated") and grey:
        hw = (64, 128)                                  # the large sizes are covered in colour; keeps the suite quick
    _both(_pattern(kind, *hw, grey), 75)


def test_feature_maps_in_mode_l_equal_pil_and_cv2():
    from oracle import raster_oracle as R
    lm, sh = R.make_landmarks(2, (256, 256), seed=3, spill=0.1)
    for i in range(2):
        fm = R.feature_map_tensor(lm[i], (256, 256), sh[i])
        _both((np.asarray(fm)[0] * 255.0).astype(np.uint8), 75)        # demo.py:270: np.uint8(map * 255)


def test_golden_files():
    cases = json.load(open(os.path.join(GOLDEN, "cases.json")))["cases"]
    assert cases
    for c in cases:
        img = np.random.default_rng(c["seed"]).integers(0, 256, c["shape"]).astype(np.uint8)
        assert J.encode(img, c["quality"]) == open(os.path.join(GOLDEN, c["file"]), "rb").read(), c["file"]


def test_quantize_divide_equals_libjpeg_turbo_reciprocal():
    x = np.arange(-32768, 32768)
    for q in range(1, 256):
        d = 8 * q
        want = np.where(x < 0, -((np.abs(x) + d // 2) // d), (np.abs(x) + d // 2) // d)
        assert np.array_equal(J.quantize_reciprocal(x, d), want), q


def test_stages_compose_to_the_file():
    img = _pattern("noise", 32, 48, False, seed=9)
    y, cb, cr = J.rgb_to_ycc(img)
    assert J.downsample_h2v2(cb).shape == (16, 24)
    zz, comp = J.scan_blocks(img, 75)
    assert zz.shape == (6 * 2 * 3, 64) and list(comp[:6]) == [0, 0, 0, 0, 1, 2]
    bits = J.block_bits(zz, comp)
    scan = J.scan_bytes(zz, comp)
    assert (int(bits.sum()) + 7) // 8 == len(scan) - scan.count(b"\xff\x00")
    assert J.header(32, 48, 3, 75) + scan + b"\xff\xd9" == J.encode(img, 75)


def _adversarial_blocks():
    """Sample blocks whose q100 coefficients are large and nonzero: alternating extremes and +-checkers."""
    out = []
    for seed in range(6):
        rng = np.random.default_rng(seed)
        b = rng.integers(0, 2, (16, 16)) * 255
        out.append(b)
    yy, xx = np.meshgrid(np.arange(16), np.arange(16), indexing="ij")
    out.append(((yy + xx) % 2) * 255)
    out.append(((yy // 2 + xx // 3) % 2) * 255)
    return [b.astype(np.uint8) for b in out]


def _handle():
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.lspj_create(C.byref(h), -1) == 0
    return lib, h


def test_max_bytes_bounds_the_worst_blocks():
    lib, h = _handle()
    out = C.c_size_t()
    for grey in (True, False):
        for b in _adversarial_blocks():
            img = b if grey else np.stack([b, 255 - b, b[::-1]], -1)
            img = np.tile(img, (4, 4) if grey else (4, 4, 1))             # 64 x 64
            zz, comp = J.scan_blocks(img, 100)
            bits = J.block_bits(zz, comp)
            assert bits.max() <= J.worst_block_bits()
            assert lib.lspj_max_bytes(h, 64, 64, 1 if grey else 3, C.byref(out)) == 0
            assert out.value == J.max_bytes(64, 64, 1 if grey else 3)
            assert out.value >= len(J.encode(img, 100))
            assert out.value >= len(J.header(64, 64, 1 if grey else 3, 100)) + 2 * (len(zz) * J.worst_block_bits()) // 8
    lib.lspj_destroy(h)


def test_header_declares_exactly_the_bound_symbols():
    header = open(os.path.join(ROOT, "include", "lspj.h")).read()
    declared = set(re.findall(r"^(?:int|const char\*)\s+(lspj_\w+)\s*\(", header, flags=re.M))
    assert declared == set(_lib.symbols("lspj"))
    lib = _lib.load()
    for name in declared:
        assert getattr(lib, name).argtypes is not None


def test_create_refuses_a_device_below_minus_one():
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.lspj_create(C.byref(h), -2) == -1 and b"device" in lib.lspj_last_error()
    assert lib.lspj_create(None, -1) == -1 and lib.lspj_last_error() == b"null argument"


def test_bad_arguments_are_refused_with_the_modules_message():
    lib, h = _handle()
    sz = C.c_size_t()
    cases = [
        (lambda: lib.lspj_max_bytes(h, 24, 32, 3, C.byref(sz)), b"multiples of 16"),
        (lambda: lib.lspj_max_bytes(h, 32, 65536, 3, C.byref(sz)), b"multiples of 16"),
        (lambda: lib.lspj_max_bytes(h, 0, 32, 3, C.byref(sz)), b"multiples of 16"),
        (lambda: lib.lspj_max_bytes(h, 32, 32, 2, C.byref(sz)), b"components"),
        (lambda: lib.lspj_max_bytes(h, 32, 32, 3, None), b"null argument"),
        (lambda: lib.lspj_max_bytes(h, 65520, 65520, 3, C.byref(sz)), b"2^30"),
        (lambda: lib.lspj_workspace_bytes(h, -1, 32, 32, 3, C.byref(sz)), b"n must be"),
        (lambda: lib.lspj_encode(h, 256, 1, 32, 32, 3, 0, 256, 10 ** 6, 256, 256, 10 ** 9, None), b"quality"),
        (lambda: lib.lspj_encode(h, 256, 1, 32, 32, 3, 101, 256, 10 ** 6, 256, 256, 10 ** 9, None), b"quality"),
        (lambda: lib.lspj_encode(h, 256, 1, 32, 32, 3, 75, 256, 100, 256, 256, 10 ** 9, None), b"out_stride"),
        (lambda: lib.lspj_encode(h, 256, 1, 32, 32, 3, 75, 256, 10 ** 6, 256, 256, 1, None), b"workspace"),
        (lambda: lib.lspj_encode(h, None, 1, 32, 32, 3, 75, 256, 10 ** 6, 256, 256, 10 ** 9, None), b"null buffer"),
        (lambda: lib.lspj_encode(h, 258, 1, 32, 32, 3, 75, 256, 10 ** 6, 256, 256, 10 ** 9, None), b"aligned"),
        (lambda: lib.lspj_encode(h, 256, -1, 32, 32, 3, 75, 256, 10 ** 6, 256, 256, 10 ** 9, None), b"n must be"),
        (lambda: lib.lspj_encode(None, 256, 1, 32, 32, 3, 75, 256, 10 ** 6, 256, 256, 10 ** 9, None), b"null handle"),
    ]
    for call, msg in cases:
        assert call() == -1, msg                                         # LSPG_EINVAL
        assert msg in lib.lspj_last_error(), (msg, lib.lspj_last_error())
    lib.lspj_destroy(h)


def test_encoding_on_a_host_only_handle_needs_the_device():
    lib, h = _handle()
    assert lib.lspj_encode(h, 256, 1, 32, 32, 3, 75, 256, 10 ** 6, 256, 256, 10 ** 9, None) == -2   # LSPG_ENODEV
    assert b"host-only handle" in lib.lspj_last_error()
    sz = C.c_size_t()
    assert lib.lspj_workspace_bytes(h, 3, 32, 32, 3, C.byref(sz)) == 0 and sz.value > 0
    lib.lspj_destroy(h)
