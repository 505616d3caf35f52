"""Generate tests/golden/lle/*.npz by running the UNMODIFIED KNN / LLE functions of the reference.  TEST INFRASTRUCTURE.

Run in the build container (needs /root/reference):  ``python oracle/make_golden_lle.py``

``funcs/utils.py`` cannot be imported here (it pulls librosa in through ``audio_funcs``), so ``KNN_with_torch`` (:100-116),
``solve_LLE_projection`` (:121-157) and ``compute_LLE_projection_all_frame`` (:171-179) are lifted out of the file with
``ast`` at run time and executed unchanged (oracle/lle_oracle.py ``reference_functions``; nothing is copied into this
repository).  The restatement in oracle/lle_oracle.py is asserted bit-equal to them while generating.

Stored per case: the seeds and sizes (the database and queries are regenerated from them, and the sha256 of the
regenerated database bytes is stored to prove it), ``ind`` and ``w`` of every row, ``feat_fuse`` of every row (every 8th
row for the 1374-row case and every 2nd for the K = 32 case, to keep the files small), and the largest |fp32 reference - float64 truth| of ``w`` and
``feat_fuse`` seen on the case.  The files live in tests/golden/lle/, apart from the generator goldens one level up.
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import lle_oracle as L  # noqa: E402

# (name, queries n, database rows N, K, database seed, query seed, feat_fuse row stride)
CASES = [
    ("lle_1374x10k_k10", 1374, 10000, 10, 1, 2, 8),     # the shipped clip (11.5 s, two mel frames per video frame)
    ("lle_37x700_k2", 37, 700, 2, 3, 4, 1),             # ragged: neither size is a multiple of a tile
    ("lle_64x2k_k1", 64, 2000, 1, 5, 6, 1),             # K = 1: w = 1, feat_fuse = the nearest row
    ("lle_200x3k_k32", 200, 3000, 32, 7, 8, 2),         # the largest K the CUDA path takes
]
DIM = 512


def main() -> None:
    out_dir = os.path.join(os.path.dirname(HERE), "tests", "golden", "lle")
    os.makedirs(out_dir, exist_ok=True)
    ref = L.reference_functions()
    for name, n, N, K, db_seed, q_seed, stride in CASES:
        db = L.make_database(N, DIM, db_seed)
        q = L.make_queries(n, DIM, q_seed, db)
        ind = ref["KNN_with_torch"](q, db, K=K)
        assert np.array_equal(ind, L.knn_with_torch(q, db, K)), name
        w, fuse = ref["compute_LLE_projection_all_frame"](q, db, ind, n)
        w2, fuse2 = L.compute_lle_projection_all(q, db, ind)
        assert ind.dtype == np.int64 and w.dtype == np.float64 and fuse.dtype == np.float32
        assert np.array_equal(w, w2) and np.array_equal(fuse, fuse2), name
        tw, tf, cond = L.lle_truth(q, db, ind)
        err_w, err_f = float(np.abs(w - tw).max()), float(np.abs(fuse - tf).max())
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), n=n, N=N, K=K, dim=DIM, db_seed=db_seed, q_seed=q_seed,
                            db_sha256=L.sha256(db), ind=ind, w=w, fuse_rows=np.arange(0, n, stride), feat_fuse=fuse[::stride],
                            err_w=err_w, err_fuse=err_f)
        print(f"{name}: max|w - truth| {err_w:.3g}, max|feat_fuse - truth| {err_f:.3g}, max cond(G) {cond.max():.3g}")


if __name__ == "__main__":
    main()
