"""The H.264 restatement (oracle/h264_oracle.py) on the host: every stream it writes decodes, through the libavcodec that
opencv-python bundles (tests/libavcodec.py), to exactly its reconstruction; its bound holds on adversarial content; a
stream cut into pushes equals the whole clip; the host-only checks of include/lspv.h; and the H.264 AVI container."""
import ctypes as C
import os
import re
import struct

import numpy as np
import pytest

import avi_reader
import libavcodec
from h264_cases import CASES, case_id, clip
from livespeechportraits_b200 import _lib
from livespeechportraits_b200.video import MjpegAviWriter
from oracle import h264_oracle as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_decoder = pytest.mark.skipif(not libavcodec.available(), reason="opencv-python's libavcodec 62 is not installed")


def _decodes_to_reconstruction(aus, recs):
    dec = libavcodec.decode(aus)
    assert len(dec) == len(recs)
    for i, (d, r) in enumerate(zip(dec, recs)):
        for k in range(3):
            assert np.array_equal(d[k], r[k]), (i, "YUV"[k], np.argwhere(d[k] != r[k])[:3])


@needs_decoder
@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_libavcodec_decodes_the_oracle_stream_to_its_reconstruction(case):
    kind, h, w, qp, gop, search, n = case
    aus, idrs, recs, state = H.encode(clip(kind, n, h, w, seed=h + w + qp), qp=qp, gop=gop, search=search)
    assert idrs == [i % gop == 0 for i in range(n)] and state.frame == n
    _decodes_to_reconstruction(aus, recs)
    assert all(len(a) <= H.max_bytes(h, w) for a in aus)


def test_static_clips_skip_every_p_macroblock():
    aus, _, _, _ = H.encode(clip("static", 4, 48, 32), qp=26, gop=60, search=4)
    # once the reference has settled: start code, NAL header, slice header and one mb_skip_run of all 6 macroblocks
    assert [len(a) for a in aus[2:]] == [8, 8]


def test_far_motion_is_coded_within_the_search_range():
    frames = clip("far", 3, 64, 80)
    src = [H.to_yuv(f) for f in frames]
    mv = H.motion_search(src[1][0], src[0][0], 26, 4)
    assert np.abs(mv).max() <= 4


@pytest.mark.parametrize("gop", [1, 60])
def test_the_bound_holds_on_adversarial_content_at_qp_0(gop):
    yy, xx = np.mgrid[0:64, 0:64]
    rng = np.random.default_rng(3)
    frames = [rng.integers(0, 256, (64, 64, 3), dtype=np.uint8),
              (((yy + xx) % 2) * 255).astype(np.uint8).repeat(3).reshape(64, 64, 3),
              np.where((yy // 16) % 2 == 0, 0, 255).astype(np.uint8).repeat(3).reshape(64, 64, 3),
              rng.integers(0, 2, (64, 64, 3)).astype(np.uint8) * 255,
              255 - rng.integers(0, 2, (64, 64, 3)).astype(np.uint8) * 255]
    aus, _, recs, _ = H.encode(frames, qp=0, gop=gop, search=3)
    bound = H.max_bytes(64, 64)
    assert max(len(a) for a in aus) <= bound
    # the levels that meet the clamp are the DC ones of a 0 -> 255 edge: the bound counts them at their longest
    assert H.worst_mb_bits(16) * 16 // 8 < bound
    if libavcodec.available():
        _decodes_to_reconstruction(aus, recs)


def test_dc_levels_beyond_2063_are_clamped_and_still_decode():
    img = np.zeros((32, 32, 3), np.uint8)
    img[16:] = 255                                   # bottom row of macroblocks predicted from black: DC level ~6500
    src = H.to_yuv(img)
    rec = [np.zeros_like(p) for p in src]
    mbs = [[H.intra_mb(src, rec, mx, my, 0) for mx in range(2)] for my in range(2)]
    assert max(int(np.abs(m.dc).max()) for row in mbs for m in row) == H.LEVEL_MAX
    if libavcodec.available():
        aus, _, recs, _ = H.encode([img], qp=0, gop=1)
        _decodes_to_reconstruction(aus, recs)


@pytest.mark.parametrize("push", [1, 7, 32])
def test_pushes_equal_the_whole_clip(push):
    frames = clip("smooth", 40, 32, 48, seed=4)
    whole, _, _, _ = H.encode(frames, qp=28, gop=16, search=4)
    state, parts = None, []
    for at in range(0, 40, push):
        aus, _, _, state = H.encode(frames[at:at + push], qp=28, gop=16, search=4, state=state)
        parts += aus
    assert parts == whole


def test_levels_of_table_a1():
    assert H.level_idc(16, 16, 60) == 10
    assert H.level_idc(512, 512, 60) == 31
    assert H.level_idc(512, 512, 25) == 30
    assert H.level_idc(1024, 1024, 60) == 40 and H.level_idc(1024, 1024, 50) == 32
    assert H.level_idc(1088, 1920, 30) == 40
    assert H.level_idc(16, 2048, 1) == 31                 # 128 macroblocks wide needs 8 MaxFS >= 128^2
    assert H.level_idc(4096, 4096, 60) == 60 and H.level_idc(8192, 8192, 1) == 0


def _prefix_free(codes):
    words = [format(c, f"0{n}b") for n, c in codes]
    assert len(set(words)) == len(words)
    for a in words:
        for b in words:
            assert a == b or not b.startswith(a), (a, b)
    return sum(2.0 ** -len(w) for w in words)


def test_the_cavlc_tables_are_complete_prefix_codes():
    for k in range(4):
        entries = [(H._CT_LEN[k][4 * tc + t1], H._CT_CODE[k][4 * tc + t1]) for tc in range(17) for t1 in range(min(tc, 3) + 1)]
        kraft = _prefix_free(entries)
        assert kraft <= 1.0 and (k == 3 or kraft > 0.99), (k, kraft)
    assert _prefix_free([(H._CDC_LEN[4 * tc + t1], H._CDC_CODE[4 * tc + t1]) for tc in range(5)
                         for t1 in range(min(tc, 3) + 1)]) <= 1.0
    for tc in range(1, 16):
        assert 0.99 < _prefix_free(list(zip(H._TZ_LEN[tc - 1], H._TZ_CODE[tc - 1]))) <= 1.0, tc
        assert len(H._TZ_LEN[tc - 1]) == 17 - tc
    for tc in range(1, 4):
        assert _prefix_free(list(zip(H._CTZ_LEN[tc - 1], H._CTZ_CODE[tc - 1]))) == 1.0
    for z in range(1, 8):
        assert _prefix_free(list(zip(H._RB_LEN[z - 1], H._RB_CODE[z - 1]))) <= 1.0
    assert sorted(H.INTER_CBP) == list(range(48))


def test_emulation_prevention():
    assert H.emulation_prevention(bytes([0, 0, 0, 0, 1, 0, 0, 2, 0, 0, 4])) == \
        bytes([0, 0, 3, 0, 0, 3, 1, 0, 0, 3, 2, 0, 0, 4])


# ---- include/lspv.h on a host-only handle ------------------------------------------------------------------------------

def _handle(qp=26, gop=60, search=16, fps=60):
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.lspv_create(C.byref(h), qp, gop, search, fps, -1) == 0
    return lib, h


def test_header_declares_exactly_the_bound_symbols():
    header = open(os.path.join(ROOT, "include", "lspv.h")).read()
    declared = set(re.findall(r"^(?:int|const char\*)\s+(lspv_\w+)\s*\(", header, flags=re.M))
    assert declared == set(_lib.symbols("lspv"))
    lib = _lib.load()
    for name in declared:
        assert getattr(lib, name).argtypes is not None


def test_max_bytes_equals_the_oracle_bound():
    lib, h = _handle()
    out = C.c_size_t()
    for hw in [(16, 16), (48, 32), (512, 512), (512, 1024), (1088, 1920)]:
        assert lib.lspv_max_bytes(h, *hw, C.byref(out)) == 0
        assert out.value == H.max_bytes(*hw), hw
        assert lib.lspv_state_bytes(h, *hw, C.byref(out)) == 0 and out.value == 256 + hw[0] * hw[1] * 3 // 2
        assert lib.lspv_workspace_bytes(h, *hw, C.byref(out)) == 0 and out.value > 0
    lib.lspv_destroy(h)


def test_bad_arguments_are_refused_with_the_modules_message():
    lib = _lib.load()
    h = C.c_void_p()
    for args, msg in [((52, 60, 16, 60), b"qp"), ((-1, 60, 16, 60), b"qp"), ((26, 0, 16, 60), b"gop"),
                      ((26, 60, 65, 60), b"search"), ((26, 60, 16, 0), b"fps")]:
        assert lib.lspv_create(C.byref(h), *args, -1) == -1 and msg in lib.lspv_last_error()
    assert lib.lspv_create(C.byref(h), 26, 60, 16, 60, -2) == -1 and b"device" in lib.lspv_last_error()
    assert lib.lspv_create(None, 26, 60, 16, 60, -1) == -1 and lib.lspv_last_error() == b"null argument"
    lib, h = _handle()
    sz = C.c_size_t()
    big = 10 ** 9
    cases = [
        (lambda: lib.lspv_max_bytes(h, 24, 32, C.byref(sz)), b"multiples of 16"),
        (lambda: lib.lspv_max_bytes(h, 32, 65536, C.byref(sz)), b"multiples of 16"),
        (lambda: lib.lspv_max_bytes(h, 32, 32, None), b"null argument"),
        (lambda: lib.lspv_max_bytes(h, 8192, 8192, C.byref(sz)), b"level"),
        (lambda: lib.lspv_encode(h, 256, 1, 32, 32, 2, 0, 256, 256, big, 256, 256, 256, big, None), b"components"),
        (lambda: lib.lspv_encode(h, 256, 1, 32, 32, 3, -1, 256, 256, big, 256, 256, 256, big, None), b"f0"),
        (lambda: lib.lspv_encode(h, 256, -1, 32, 32, 3, 0, 256, 256, big, 256, 256, 256, big, None), b"n must be"),
        (lambda: lib.lspv_encode(h, 256, 1, 32, 32, 3, 0, 256, 256, 100, 256, 256, 256, big, None), b"out_stride"),
        (lambda: lib.lspv_encode(h, 256, 1, 32, 32, 3, 0, 256, 256, big, 256, 256, 256, 1, None), b"workspace"),
        (lambda: lib.lspv_encode(h, None, 1, 32, 32, 3, 0, 256, 256, big, 256, 256, 256, big, None), b"null buffer"),
        (lambda: lib.lspv_encode(h, 256, 1, 32, 32, 3, 0, 256, 256, big, 256, 256, 258, big, None), b"aligned"),
        (lambda: lib.lspv_encode(None, 256, 1, 32, 32, 3, 0, 256, 256, big, 256, 256, 256, big, None), b"null handle"),
    ]
    for call, msg in cases:
        assert call() == -1, msg                                         # LSPG_EINVAL
        assert msg in lib.lspv_last_error(), (msg, lib.lspv_last_error())
    assert lib.lspv_encode(h, 256, 1, 32, 32, 3, 0, 256, 256, big, 256, 256, 256, big, None) == -2   # LSPG_ENODEV
    assert b"host-only handle" in lib.lspv_last_error()
    lib.lspv_destroy(h)


# ---- the H.264 AVI ----------------------------------------------------------------------------------------------------

def _h264_avi(path, aus, idrs, audio=None):
    with MjpegAviWriter(path, (64, 48), 25, None if audio is None else 8000, fourcc="H264") as w:
        if audio is not None:
            w.write_audio(audio)
        for a, k in zip(aus, idrs):
            w.write_frame(a, keyframe=k)


def test_h264_avi_flags_keyframes_only_on_idrs(tmp_path):
    aus, idrs, _, _ = H.encode(clip("smooth", 9, 48, 64), qp=30, gop=4, search=4)
    path = str(tmp_path / "v.avi")
    _h264_avi(path, aus, idrs, np.zeros(8000, np.float32))
    r = avi_reader.read(path)
    assert r["strh"][0][1] == b"H264" and r["strf"][0][16:20] == b"H264"
    assert r["data"](b"00dc") == aus
    assert [bool(flags & 0x10) for cid, flags, _, _ in r["idx1"] if cid == b"00dc"] == idrs
    buf = open(path, "rb").read()
    (chunk_id, entries), = [e for e in r["indx"] if e[0] == b"00dc"]
    keys = []
    for off, _, _ in entries:
        n = struct.unpack_from("<I", buf, off + 12)[0]
        keys += [not struct.unpack_from("<II", buf, off + 32 + 8 * i)[1] >> 31 for i in range(n)]
    assert keys == idrs


def test_cv2_reads_every_frame_of_an_h264_avi(tmp_path):
    cv2 = pytest.importorskip("cv2")
    aus, idrs, recs, _ = H.encode(clip("translate", 12, 48, 64), qp=24, gop=5, search=8)
    path = str(tmp_path / "v.avi")
    _h264_avi(path, aus, idrs)
    cap = cv2.VideoCapture(path)
    assert cap.isOpened()
    frames = []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        frames.append(f)
    cap.release()
    assert len(frames) == 12 and frames[0].shape == (48, 64, 3)
    # cv2 converts to BGR with its own arithmetic: compare its luma with the reconstruction's loosely
    for f, r in zip(frames, recs):
        y = (0.257 * f[:, :, 2] + 0.504 * f[:, :, 1] + 0.098 * f[:, :, 0] + 16)
        assert np.abs(y - r[0]).mean() < 6


def test_the_default_fourcc_writes_the_bytes_it_always_wrote(tmp_path):
    import hashlib
    rng = np.random.default_rng(7)
    path = str(tmp_path / "m.avi")
    with MjpegAviWriter(path, (32, 16), 25, audio_rate=8000, audio_channels=2, audio_format="s16",
                        segment_bytes=4096) as w:
        w.write_audio(rng.integers(-3000, 3000, (8000, 2), dtype=np.int16))
        for i in range(30):
            w.write_frame(bytes(rng.integers(0, 256, 100 + 37 * i, dtype=np.uint8)))
    # the file MjpegAviWriter wrote before it took a fourcc, with these seeded frames and audio
    assert hashlib.sha256(open(path, "rb").read()).hexdigest() == \
        "191bc765ad55c41910e79ccce52056835bb5ca28fb39601b03d8cdb79e8ecb1f"


def test_the_goldens_are_the_oracles_streams():
    import json
    golden = os.path.join(ROOT, "tests", "golden", "h264")
    for c in json.load(open(os.path.join(golden, "cases.json"))):
        frames = clip(c["kind"], c["frames"], c["height"], c["width"], seed=c["seed"])
        aus, _, recs, _ = H.encode(frames, qp=c["qp"], gop=c["gop"], search=c["search"])
        assert b"".join(aus) == open(os.path.join(golden, c["name"] + ".h264"), "rb").read(), c["name"]
        planes = np.load(os.path.join(golden, c["name"] + ".npz"))             # libavcodec's decoding, stored
        for i, r in enumerate(recs):
            for k, p in enumerate("yuv"):
                assert np.array_equal(r[k], planes[f"{p}{i}"]), (c["name"], i, p)
