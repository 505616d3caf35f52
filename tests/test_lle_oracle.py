"""Row N5 (SURVEY.md 8f), CPU part: the oracle of the APC manifold projection (oracle/lle_oracle.py) pinned against the
golden vectors generated from the reference's KNN_with_torch / compute_LLE_projection_all_frame and, where the reference
checkout exists, against those functions themselves; the C ABI's argument checking on a host-only handle; install() on a
stand-in funcs.utils module."""
import ctypes as C
import inspect
import os
import sys
import types

import numpy as np
import pytest
import torch

from livespeechportraits_b200 import _lib, manifold
from oracle import lle_oracle as L

GOLD_DIR = os.path.join(os.path.dirname(__file__), "golden", "lle")
GOLDENS = ["lle_1374x10k_k10", "lle_37x700_k2", "lle_64x2k_k1", "lle_200x3k_k32"]


def _golden(name):
    g = np.load(os.path.join(GOLD_DIR, name + ".npz"))
    db = L.make_database(int(g["N"]), int(g["dim"]), int(g["db_seed"]))
    q = L.make_queries(int(g["n"]), int(g["dim"]), int(g["q_seed"]), db)
    return g, db, q


def test_test_data_are_deterministic_and_in_range():
    a, b = L.make_database(1200, 64, 3), L.make_database(1200, 64, 3)
    assert a.dtype == np.float32 and a.shape == (1200, 64) and np.array_equal(a, b)
    assert np.abs(a).max() < 1.0
    q = L.make_queries(50, 64, 4, a)
    assert q.dtype == np.float32 and np.array_equal(q, L.make_queries(50, 64, 4, a))
    assert not np.array_equal(a, L.make_database(1200, 64, 4))


@pytest.mark.parametrize("name", GOLDENS)
def test_restatement_matches_the_goldens(name):
    """Written by oracle/make_golden_lle.py from the UNMODIFIED reference functions, where the restatement was bit-equal
    to them.  The database is regenerated bit for bit (sha256).  fp32 BLAS kernels differ between CPU models, so here
    the indices follow the KNN band rule and w / feat_fuse stay within twice the recorded fp32-vs-float64 error."""
    g, db, q = _golden(name)
    assert L.sha256(db) == str(g["db_sha256"])
    k = int(g["K"])
    ind = L.knn_with_torch(q, db, k)
    L.check_knn_band(ind, q, db, k, g["ind"])
    L.check_knn_band(g["ind"], q, db, k)
    w, fuse = L.compute_lle_projection_all(q, db, g["ind"])
    assert w.dtype == np.float64 and fuse.dtype == np.float32
    err_w, err_f = float(g["err_w"]), float(g["err_fuse"])
    assert np.abs(w - g["w"]).max() <= 2 * err_w + 1e-7
    assert np.abs(fuse[g["fuse_rows"]] - g["feat_fuse"]).max() <= 2 * err_f + 1e-7


@pytest.mark.parametrize("name", GOLDENS)
def test_float64_truth_vs_fp32_reference_within_recorded_bounds(name):
    g, db, q = _golden(name)
    tw, tf, cond = L.lle_truth(q, db, g["ind"])
    assert np.abs(g["w"] - tw).max() <= float(g["err_w"]) + 1e-12
    assert np.abs(g["feat_fuse"] - tf[g["fuse_rows"]]).max() <= float(g["err_fuse"]) + 1e-12
    assert float(g["err_fuse"]) <= 1e-5 and np.isfinite(cond).all()
    if int(g["K"]) == 1:
        assert (g["w"] == 1).all() and np.array_equal(g["feat_fuse"], db[g["ind"][g["fuse_rows"], 0]])


@pytest.mark.skipif(not L.reference_available(), reason="reference checkout not present on this machine")
@pytest.mark.parametrize("name", GOLDENS)
def test_restatement_is_bit_equal_to_the_live_reference(name):
    ref = L.reference_functions()
    g, db, q = _golden(name)
    k = int(g["K"])
    ind = ref["KNN_with_torch"](q, db, K=k)
    assert np.array_equal(ind, L.knn_with_torch(q, db, k))
    w, fuse = ref["compute_LLE_projection_all_frame"](q, db, ind, q.shape[0])
    w2, fuse2 = L.compute_lle_projection_all(q, db, ind)
    assert np.array_equal(w, w2) and np.array_equal(fuse, fuse2)
    v, f = ref["solve_LLE_projection"](q[0], db[ind[0]])
    v2, f2 = L.solve_lle_projection(q[0], db[ind[0]])
    assert np.array_equal(v, v2) and np.array_equal(f, f2) and f.dtype == f2.dtype


def test_duplicated_row_is_singular_in_the_restatement():
    db, q, src, dst = L.make_singular_case()
    ind = L.knn_with_torch(q, db, 10)
    assert set(ind[0, :2].tolist()) == {src, dst}
    with pytest.raises(np.linalg.LinAlgError):
        L.compute_lle_projection_all(q, db, ind)
    if L.reference_available():
        ref = L.reference_functions()
        with pytest.raises(np.linalg.LinAlgError):
            ref["compute_LLE_projection_all_frame"](q, db, ind, q.shape[0])


def test_host_only_handle_argument_checks():
    lib = _lib.load()
    h = C.c_void_p()
    for dim in (0, 500, 1056, -32):
        assert lib.lspm_create(C.byref(h), dim, -1) == -1, dim
    assert lib.lspm_create(None, 512, -1) == -1
    if not torch.cuda.is_available():
        assert lib.lspm_create(C.byref(h), 512, 0) == -2                  # no device, no fallback
    assert lib.lspm_create(C.byref(h), 512, -1) == 0
    try:
        size = C.c_size_t()
        assert lib.lspm_workspace_bytes(h, 1374, 10, C.byref(size)) == 0 and size.value > 0
        for n, k in ((0, 10), (-3, 10), (10, 0), (10, 33)):
            assert lib.lspm_workspace_bytes(h, n, k, C.byref(size)) == -1, (n, k)
        assert lib.lspm_workspace_bytes(h, 10, 10, None) == -1
        assert lib.lspm_workspace_bytes(h, 1374, 10, C.byref(size)) == 0
        need = size.value
        buf = (C.c_float * 16)()
        p = C.cast(buf, C.c_void_p)
        knn = lambda feats, n, k, out, ws, nbytes: lib.lspm_knn(h, feats, n, k, out, None, ws, nbytes, None)   # noqa: E731
        assert knn(p, 1374, 0, p, p, need) == -1
        assert knn(p, 1374, 33, p, p, need) == -1
        assert knn(p, 0, 10, p, p, need) == -1
        assert knn(None, 1374, 10, p, p, need) == -1
        assert knn(p, 1374, 10, None, p, need) == -1
        assert knn(p, 1374, 10, p, None, need) == -1
        assert knn(p, 1374, 10, p, p, need - 1) == -1 and b"workspace" in lib.lspm_last_error()
        assert knn(p, 1374, 10, p, p, need) == -2 and b"no CPU path" in lib.lspm_last_error()
        proj = lambda feats, n, ind, k: lib.lspm_project(h, feats, n, ind, k, 1.0, None, None, None, None, None)   # noqa: E731
        assert proj(p, 0, p, 10) == -1
        assert proj(p, 4, p, 0) == -1 and proj(p, 4, p, 33) == -1
        assert proj(None, 4, p, 10) == -1 and proj(p, 4, None, 10) == -1
        assert proj(p, 4, p, 10) == -2 and b"no CPU path" in lib.lspm_last_error()
        db = np.zeros((4, 512), np.float32)
        assert lib.lspm_load_database(h, db.ctypes.data, 0) == -1
        assert lib.lspm_load_database(h, db.ctypes.data, 1 << 31) == -1
        assert lib.lspm_load_database(h, None, 4) == -1
        assert lib.lspm_load_database(h, db.ctypes.data, 4) == -2 and b"no CPU path" in lib.lspm_last_error()
    finally:
        assert lib.lspm_destroy(h) == 0
    assert lib.lspm_destroy(None) == 0


def test_python_layer_refuses_the_cpu():
    with pytest.raises(RuntimeError, match="no CPU path"):
        manifold.ManifoldProjector(np.zeros((4, 512), np.float32), device=torch.device("cpu"))


def test_install_replaces_both_functions_with_the_reference_signatures():
    mod = types.ModuleType("lspm_stand_in_utils")
    mod.KNN_with_torch = L.knn_with_torch
    mod.compute_LLE_projection_all_frame = L.compute_lle_projection_all
    sys.modules[mod.__name__] = mod
    try:
        manifold.install(mod.__name__)
        assert mod.KNN_with_torch is manifold.KNN_with_torch
        assert mod.compute_LLE_projection_all_frame is manifold.compute_LLE_projection_all_frame
        assert str(inspect.signature(mod.KNN_with_torch)) == "(feats, feat_database, K=10)"
        assert str(inspect.signature(mod.compute_LLE_projection_all_frame)) == "(feats, feat_database, ind, nframe)"
        if L.reference_available():
            ref = L.reference_functions()
            for fn in ("KNN_with_torch", "compute_LLE_projection_all_frame"):
                assert inspect.signature(getattr(mod, fn)) == inspect.signature(ref[fn]), fn
        # float32 only, as APC output is (the reference's own matmul fails on mixed dtypes)
        db = np.zeros((8, 512), np.float32)
        with pytest.raises(TypeError):
            mod.KNN_with_torch(np.zeros((2, 512)), db, K=2)
        with pytest.raises(TypeError):
            mod.compute_LLE_projection_all_frame(np.zeros((2, 512), np.float32), db.astype(np.float64), np.zeros((2, 2), np.int64), 2)
        with pytest.raises(IndexError):
            mod.compute_LLE_projection_all_frame(np.zeros((2, 512), np.float32), db, np.full((2, 2), 8), 2)
        if not torch.cuda.is_available():
            with pytest.raises(RuntimeError, match="no CPU path"):
                mod.KNN_with_torch(np.zeros((2, 512), np.float32), db, K=2)
    finally:
        sys.modules.pop(mod.__name__, None)
