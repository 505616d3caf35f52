"""Row N7 (SURVEY.md 8f), CPU part: the oracle of the landmark post-processing (oracle/landmark_oracle.py) pinned against
the golden vectors generated from demo.py's stage-5 statements; its reflect-rule filter against scipy; ``amp_table``
against ``mouth_pts_AMP``; the kernel emulation within ``error_bound`` and each planted defect outside it; the C ABI's
declared symbols and its argument checking on a host-only handle."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest
import torch
from scipy.ndimage import gaussian_filter1d

from livespeechportraits_b200 import _lib, landmarks as L
from oracle import landmark_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD_DIR = os.path.join(os.path.dirname(__file__), "golden", "landmarks")
GOLDENS = ["may_672", "obama1_672", "xy_200", "lowermore_200", "mouth_sigma0_150", "head_longer_300_340",
           "feat_longer_340_300", "no_crossing_200", "n1", "n2", "n7", "n41", "pad_200"]
KEYS = (("pred_landmarks", "landmarks"), ("pred_shoulders", "shoulders"), ("final_pts3d", "final_pts3d"),
        ("pred_headpose", "pred_headpose"))


def golden(name):
    """(pred_Feat, pred_Head, identity, params, image_pad, reference outputs) of one golden case."""
    g = np.load(os.path.join(GOLD_DIR, name + ".npz"))
    ident = {k: g["id_" + k] for k in O.IDENTITY_KEYS}
    ident["scale"] = np.float64(ident["scale"])
    pad = tuple(int(v) for v in g["image_pad"]) or None
    return g["pred_Feat"], g["pred_Head"], ident, json.loads(str(g["params"])), pad, {k: g[k] for k, _ in KEYS}


@pytest.mark.parametrize("name", GOLDENS)
def test_restatement_matches_the_goldens_bit_for_bit(name):
    feat, head, ident, prm, pad, ref = golden(name)
    got = O.stage5(feat, head, ident, prm, image_pad=pad)
    n = min(len(feat), len(head))
    for k, _ in KEYS:
        assert np.array_equal(got[k][:n], ref[k]), k


@pytest.mark.parametrize("n", [1, 2, 7, 40, 41, 100, 672])
@pytest.mark.parametrize("sigma", [1, 1.5, 5, 10])
def test_reflect_filter_matches_scipy(n, sigma):
    x = np.random.default_rng(n).normal(0, 1, (n, 5)) + 3
    ref = gaussian_filter1d(x, sigma, axis=0)
    assert np.allclose(O.gauss_reflect(x, sigma), ref, rtol=1e-12, atol=0)


@pytest.mark.parametrize("method,paras", [("XY", [1.8, 2.2]), ("XYZ", [2, 2, 2]), ("XYZ", [1.5, 0.5, 3]),
                                          ("LowerMore", [1.2, 1.6, 1.0, 2.0, 2.4, 1.5])])
def test_amp_table_equals_mouth_pts_amp(method, paras):
    x = np.random.default_rng(3).normal(0, 1, (50, 73, 3))
    ref = O.mouth_pts_AMP(x.copy(), True, method, paras)
    got = x.copy()
    got[:, 46:64] *= L.amp_table(method, paras)
    assert np.array_equal(got, ref)
    if O.reference_available():
        live = O.reference_functions().mouth_pts_AMP(x.copy(), True, method, paras)
        assert np.array_equal(live, ref)


def test_amp_table_refusals():
    for method in ("delta", "CloseSmall"):
        with pytest.raises(NotImplementedError):
            L.amp_table(method, [1, 1, 1, 1, 1, 1])
    for method in ("xyz", "", "Lower"):
        with pytest.raises(ValueError):
            L.amp_table(method, [1, 1, 1])
    with pytest.raises(ValueError):
        L.amp_table("XYZ", [1, 1])


def test_head_sigma_zero_is_refused_where_scipy_divides_by_zero():
    with pytest.raises(ZeroDivisionError):
        gaussian_filter1d(np.ones((5, 3)), 0, axis=0)
    p = L.StageParams(1.5, "XYZ", [2, 2, 2], 1, 0.5, [0, 10], 0.5)
    with pytest.raises(ValueError, match="> 0"):
        L._native_params(p, None)
    with pytest.raises(ValueError):
        L.postprocess_clip(*([None] * 10), 1.5, "XYZ", [2, 2, 2], 1, 0.5, [5, 0], 0.5)


@pytest.mark.parametrize("name", GOLDENS)
def test_emulation_within_the_bound(name):
    feat, head, ident, prm, pad, ref = golden(name)
    t = O.truth(feat, head, ident, prm, pad)
    b = O.error_bound(t)
    e = O.emulate(feat, head, ident, prm, pad)
    for _, k in KEYS:
        assert (np.abs(e[k] - t[k]) <= b[k]).all(), k
    # the truth decides the lip fix as the reference does
    n = min(len(feat), len(head))
    assert np.abs(ref["final_pts3d"] - t["final_pts3d"][:n]).max() < 1e-5


@pytest.mark.parametrize("mutation,name", [("head_nframe", "head_longer_300_340"), ("sigma_swap", "may_672"),
                                           ("brow_shift", "may_672"), ("mouth_shift", "may_672"),
                                           ("no_lipfix", "may_672"), ("lipfix_two", "may_672"),
                                           ("pad_flip", "pad_200")])
def test_each_planted_defect_exceeds_the_bound(mutation, name):
    feat, head, ident, prm, pad, _ = golden(name)
    t = O.truth(feat, head, ident, prm, pad)
    b = O.error_bound(t)
    e = O.emulate(feat, head, ident, prm, pad, mutation=mutation)
    worst = max(float((np.abs(e[k] - t[k]) / b[k]).max()) for k in ("landmarks", "shoulders"))
    assert worst > 1.0, mutation


def test_header_declares_exactly_the_bound_symbols():
    header = open(os.path.join(ROOT, "include", "lspl.h")).read()
    declared = set(re.findall(r"^(?:int|const char\*)\s+(lspl_\w+)\s*\(", header, flags=re.M))
    assert declared == set(_lib.SYMBOLS_L), declared ^ set(_lib.SYMBOLS_L)
    lib = _lib.load()
    for name in _lib.SYMBOLS_L:
        getattr(lib, name)


def _native_identity(m=3):
    ident = O.make_identity(0, max(m, 1))
    keep = [np.ascontiguousarray(ident[k], np.float64) for k in ("mean_pts3d", "std_mean_pts3d", "candidate_eye_brow", "shoulder3D")]
    nid = _lib.LsplIdentity()
    nid.mean_pts3d, nid.std_mean_pts3d, nid.candidate_eye_brow, nid.shoulder3D = (a.ctypes.data for a in keep)
    nid.n_candidates = m
    nid.scale = 1.0
    return nid, keep


def test_host_only_handle_argument_checks():
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.lspl_create(None, -1) == -1
    assert lib.lspl_create(C.byref(h), -2) == -1
    if not torch.cuda.is_available():
        assert lib.lspl_create(C.byref(h), 0) == -2                       # no device, no fallback
    assert lib.lspl_create(C.byref(h), -1) == 0
    try:
        nid, keep = _native_identity(0)
        assert lib.lspl_load_identity(h, C.byref(nid)) == -1             # m = 0
        nid, keep = _native_identity(3)
        assert lib.lspl_load_identity(h, None) == -1
        assert lib.lspl_load_identity(h, C.byref(nid)) == -2 and b"no CPU path" in lib.lspl_last_error()
        size = C.c_size_t()
        assert lib.lspl_workspace_bytes(h, -1, 5, C.byref(size)) == -1
        assert lib.lspl_workspace_bytes(h, 5, 5, None) == -1
        assert lib.lspl_workspace_bytes(h, 100, 120, C.byref(size)) == 0 and size.value >= 100 * 54 * 8
        assert lib.lspl_workspace_bytes(h, 0, 120, C.byref(size)) == 0
        buf = (C.c_double * 64)()
        p = C.cast(buf, C.c_void_p)
        prm = _lib.LsplParams(feat_sigma=1.5, rot_sigma=5, trans_sigma=10)

        def run(nf=10, nh=10, stride=12, feat=p, head=p, lm=p, sh=p, params=prm):
            return lib.lspl_run(h, feat, nf, head, nh, stride, C.byref(params) if params is not None else None, lm, sh,
                                None, None, p, 512, None)
        assert run() == -2 and b"no CPU path" in lib.lspl_last_error()
        assert run(nf=-1) == -1 and run(nh=-1) == -1
        for stride in (5, 0, -6):
            assert run(stride=stride) == -1, stride
        assert run(params=None) == -1
        for rs, ts in ((0, 10), (5, 0), (-1, 10), (float("nan"), 10), (5, 1e6)):
            bad = _lib.LsplParams(feat_sigma=1.5, rot_sigma=rs, trans_sigma=ts)
            assert run(params=bad) == -1, (rs, ts)
        assert b"sigma" in lib.lspl_last_error()
        assert run(params=_lib.LsplParams(feat_sigma=-1, rot_sigma=5, trans_sigma=10)) == -1
        assert run(params=_lib.LsplParams(feat_sigma=0, rot_sigma=5, trans_sigma=10)) == -2    # 0: no mouth smoothing
        assert run(lm=None) == -1 and run(sh=None) == -1
        assert run(feat=None) == -1 and run(head=None) == -1
        assert run(nf=0, feat=None, lm=None, sh=None) == -2                # nframe 0 is valid
    finally:
        assert lib.lspl_destroy(h) == 0
    assert lib.lspl_destroy(None) == 0


def test_python_layer_refuses_the_cpu():
    ident = L.Identity(**O.make_identity(0))
    with pytest.raises(RuntimeError, match="no CPU path"):
        L.LandmarkPostprocessor(ident, device=torch.device("cpu"))
