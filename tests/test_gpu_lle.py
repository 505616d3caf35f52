"""Row N5 (SURVEY.md 8f) on the GPU: the KNN and LLE kernels of include/lspm.h against float64 truths and the fp32
oracle of funcs/utils.py (oracle/lle_oracle.py), the golden vectors generated from the reference, the installed drop-ins,
and the device chain into the head-pose loop.

KNN results are judged by the band rule of ``lle_oracle.check_knn_band``: the kernel ranks by the reference's fp32
expression |q|^2 + |d|^2 - 2 q.d, so near-ties (within 2^-20 of the norms) may order differently from exact arithmetic and
from ATen's summation order; everywhere else the result must equal the fp32 oracle's.  LLE results are judged against
the float64 solution of the same fp32 inputs (1e-6) and the fp32 reference (1e-4)."""
import functools
import types

import numpy as np
import pytest
import torch

from oracle import lle_oracle as L

pytestmark = pytest.mark.gpu
DIM = 512
DEV = torch.device("cuda", 0)


@functools.lru_cache(maxsize=4)
def _db(N, seed):
    return L.make_database(N, DIM, seed)


def _proj(db):
    from livespeechportraits_b200.manifold import ManifoldProjector
    return ManifoldProjector(db, device=DEV)


KNN_CASES = [(700, 37, 2), (700, 1, 1), (700, 1374, 32), (10000, 1374, 10), (10000, 37, 32), (10000, 1, 10),
             (10000, 1374, 1), (100000, 1374, 10), (100000, 1, 32)]


@pytest.mark.parametrize("N,n,k", KNN_CASES)
def test_knn_against_exact_distances(N, n, k):
    db = _db(N, 11)
    q = L.make_queries(n, DIM, 12 + n, db)
    ind = _proj(db).knn(q, k).cpu().numpy()
    frac = L.check_knn_band(ind, q, db, k, L.knn_with_torch(q, db, k), device=DEV)
    print(f"knn N={N} n={n} K={k}: {frac:.3f} of rows well separated, all equal to the fp32 oracle")


def test_knn_duplicate_rows_come_back_lower_index_first():
    db, q, src, dst = L.make_singular_case(700, 8, DIM)
    p = _proj(db)
    for k in (2, 10):
        ind = p.knn(q, k).cpu().numpy()
        assert ind[0, 0] == src and ind[0, 1] == dst, ind[0]
    # the same row in every slice of a larger base: the lowest index still wins
    big = _db(10000, 11).copy()
    rows = [123, 4567, 9999]
    for r in rows[1:]:
        big[r] = big[rows[0]]
    qq = np.ascontiguousarray(big[[rows[0]]])
    assert _proj(big).knn(qq, 3).cpu().numpy()[0].tolist() == rows


@pytest.mark.parametrize("N,n,k", [(10000, 1374, 10), (3000, 200, 32), (700, 37, 2), (2000, 64, 1), (3000, 200, 20)])
def test_lle_against_float64_truth_and_fp32_reference(N, n, k):
    db = _db(N, 13)
    q = L.make_queries(n, DIM, 14, db)
    ind = L.knn_with_torch(q, db, k)             # the oracle's indices: the LLE stage is checked on its own
    w, fuse, blend, status = (t.cpu().numpy() for t in _proj(db).project(q, ind, 1.0))
    assert w.dtype == np.float64 and fuse.dtype == np.float32 and status.dtype == np.int32
    assert (status == 0).all()
    tw, tf, cond = L.lle_truth(q, db, ind)
    ef = np.abs(fuse - tf).max()
    well = cond <= 1e6
    ew = np.abs(w - tw)[well].max()
    rw, rf = L.compute_lle_projection_all(q, db, ind)
    er = np.abs(fuse - rf).max()
    print(f"lle N={N} n={n} K={k}: max|fuse - truth| {ef:.3g}, max|w - truth| {ew:.3g} ({well.mean():.3f} of rows with "
          f"cond <= 1e6, max cond {cond.max():.3g}), max|fuse - fp32 reference| {er:.3g}")
    assert ef <= 1e-6 and ew <= 1e-6 and er <= 1e-4
    assert np.array_equal(blend, fuse)            # percent 1: feats * 0 + fuse * 1
    if k == 1:
        assert (w == 1.0).all() and np.array_equal(fuse, db[ind[:, 0]])


@pytest.mark.parametrize("percent", [0.0, 0.5, 1.0])
def test_blend_is_the_reference_fp32_expression(percent):
    db = _db(10000, 13)
    q = L.make_queries(300, DIM, 15, db)
    p = _proj(db)
    ind = p.knn(q, 10)
    _, fuse, blend, _ = p.project(q, ind, percent)
    fuse, blend = fuse.cpu().numpy(), blend.cpu().numpy()
    assert np.array_equal(blend, q * (1 - percent) + fuse * percent)        # demo.py:200 on float32 arrays
    assert torch.equal(p.project_features(q, 10, percent).cpu(), torch.from_numpy(blend))


def test_status_for_singular_rows_and_bad_indices():
    db, q, src, dst = L.make_singular_case(700, 8, DIM)
    p = _proj(db)
    ind = p.knn(q, 10).cpu().numpy()
    ind[3, 2] = 700                               # past the end
    ind[4, 0] = -1                                # negative
    ind[5, 5] = 1 << 40                           # far outside: must not be read through
    ind[6, 1] = ind[6, 4]                         # a neighbour twice: identical Gram rows
    w, fuse, blend, status = (t.cpu().numpy() for t in p.project(q, ind, 0.5))
    assert status.tolist() == [1, 0, 0, 2, 2, 2, 1, 0]
    bad = status != 0
    assert np.isnan(w[bad]).all() and np.isnan(fuse[bad]).all() and np.isnan(blend[bad]).all()
    assert np.isfinite(w[~bad]).all() and np.isfinite(fuse[~bad]).all()
    _, tf, _ = L.lle_truth(q[~bad], db, ind[~bad])
    assert np.abs(fuse[~bad] - tf).max() <= 1e-6


def _stand_in_module():
    import sys
    mod = types.ModuleType("lspm_test_utils")
    mod.KNN_with_torch = L.knn_with_torch
    mod.compute_LLE_projection_all_frame = lambda feats, feat_database, ind, nframe: L.compute_lle_projection_all(feats, feat_database, ind)
    sys.modules[mod.__name__] = mod
    return mod


@pytest.mark.parametrize("name", ["lle_1374x10k_k10", "lle_37x700_k2", "lle_64x2k_k1", "lle_200x3k_k32"])
def test_installed_drop_ins_reproduce_the_goldens(name):
    import os
    import sys
    from livespeechportraits_b200 import manifold
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "lle", name + ".npz"))
    db = L.make_database(int(g["N"]), int(g["dim"]), int(g["db_seed"]))
    assert L.sha256(db) == str(g["db_sha256"])
    q = L.make_queries(int(g["n"]), int(g["dim"]), int(g["q_seed"]), db)
    mod = _stand_in_module()
    try:
        manifold.install(mod.__name__)
        k = int(g["K"])
        ind = mod.KNN_with_torch(q, db, K=k)
        assert isinstance(ind, np.ndarray) and ind.dtype == np.int64 and ind.shape == (q.shape[0], k)
        L.check_knn_band(ind, q, db, k, g["ind"], device=DEV)
        w, fuse = mod.compute_LLE_projection_all_frame(q, db, g["ind"], q.shape[0])
        assert w.dtype == np.float64 and w.shape == g["w"].shape
        assert fuse.dtype == np.float32 and fuse.shape == q.shape
        assert np.abs(fuse[g["fuse_rows"]] - g["feat_fuse"]).max() <= 1e-4
        assert np.abs(w - g["w"]).max() <= 1e-4 + 2 * float(g["err_w"])
    finally:
        sys.modules.pop(mod.__name__, None)


def test_drop_in_raises_linalg_error_on_a_singular_row():
    from livespeechportraits_b200 import manifold
    db, q, _, _ = L.make_singular_case(700, 8, DIM)
    ind = manifold.KNN_with_torch(q, db, K=10)
    with pytest.raises(np.linalg.LinAlgError):
        manifold.compute_LLE_projection_all_frame(q, db, ind, q.shape[0])
    with pytest.raises(np.linalg.LinAlgError):
        L.compute_lle_projection_all(q, db, ind)


def test_device_chain_into_the_headpose_loop():
    """project_features -> view(-1, 1024) -> HeadposeGenerator.generate without leaving the device, bit for bit the
    same as passing the host copy (demo.py:200 then :211-212)."""
    from livespeechportraits_b200.headpose import HeadposeGenerator
    from oracle import a2h_oracle as A
    hopt = A.default_opt()
    nframe = 6
    db = _db(10000, 13)
    q = L.make_queries(2 * (hopt.frame_future + nframe), DIM, 16, db)
    blend = _proj(db).project_features(q, 10, 1.0)
    assert blend.is_cuda and blend.dtype == torch.float32
    gen = HeadposeGenerator(hopt, A.make_state_dict(hopt, "B", 1), device=DEV)
    noise = A.reference_noise(nframe, 12, 1, seed=0)
    pre = np.zeros(12, np.float32)
    on_device = gen.generate(blend.view(-1, 1024), pre, noise, 0.3)
    via_host = gen.generate(blend.cpu().numpy().reshape(-1, 1024), pre, noise, 0.3)
    assert on_device.shape == (nframe, 12) and torch.equal(on_device, via_host)
