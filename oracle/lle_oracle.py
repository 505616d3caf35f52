"""Oracle of the APC manifold projection (SURVEY.md 8f row N5): KNN search over the identity's APC feature base and the
LLE reconstruction of each feature row from its neighbours.  TEST INFRASTRUCTURE.

Restated from funcs/utils.py with the same torch / numpy calls and dtypes (nothing is copied):

* ``knn_with_torch``              <- ``KNN_with_torch`` (:100-116): fp32 ``|q|^2 + |d|^2 - 2 q.d`` on the host, ``topk``
* ``solve_lle_projection``        <- ``solve_LLE_projection`` (:121-157): fp32 normal equations, ``numpy.linalg.solve``
* ``compute_lle_projection_all``  <- ``compute_LLE_projection_all_frame`` (:171-179): one solve per row, ``w`` float64,
                                     ``feat_fuse`` in the dtype of ``feats``

and float64 truths to judge the CUDA kernels by: ``lle_truth`` (exact LLE in float64 of the same fp32 inputs, given the
indices) and ``exact_sqdist`` / ``exact_topk`` (float64 squared distances).

The test data are regenerated bit for bit on any machine: ``make_database`` / ``make_queries`` draw from numpy's PCG64 and
use only exactly-rounded operations (uniform draws, ``+``, ``*``, ``/``, ``abs``; no BLAS, no libm).  APC features are
outputs of the last GRU layer and lie in (-1, 1), so a smooth low-rank trajectory is squashed with ``x / (1 + |x|)``
(``np.tanh`` is vectorised differently on different CPUs and can differ in the last ulp).
"""
from __future__ import annotations

import ast
import os
from typing import Optional, Tuple

import numpy as np
import torch

REFERENCE_ROOT = os.environ.get("LSP_REFERENCE_ROOT", "/root/reference")
REF_FILE = os.path.join(REFERENCE_ROOT, "funcs", "utils.py")

_SEG = 500          # trajectory segment length (independent clips in the database)
_CHUNK = 8192       # rows generated per block; fixed, so the draw order does not depend on n


# ------------------------------------------------------------------------------------------------------------------
# Test data
# ------------------------------------------------------------------------------------------------------------------
def _uniform(rng: np.random.Generator, shape) -> np.ndarray:
    """U(-1, 1) in float64: 53 random bits scaled by a power of two, then ``* 2 - 1`` (both exact)."""
    return rng.random(shape) * 2.0 - 1.0


def make_database(n: int, dim: int = 512, seed: int = 0, rank: int = 8) -> np.ndarray:
    """[n, dim] float32 in (-1, 1): ``n / 500`` AR(1) trajectories in a ``rank``-dimensional latent space, mapped to
    ``dim`` through a random basis, plus small per-element noise, squashed by ``x / (1 + |x|)``."""
    rng = np.random.Generator(np.random.PCG64(seed))
    basis = _uniform(rng, (rank, dim))
    n_seg = -(-n // _SEG)
    z = _uniform(rng, (n_seg, rank))
    latent = np.empty((n_seg * _SEG, rank))
    for t in range(_SEG):                           # vectorised over segments; every step is a multiply and an add
        z = z * 0.95 + _uniform(rng, (n_seg, rank)) * 0.3
        latent[t::_SEG] = z
    out = np.empty((n, dim), np.float32)
    for r0 in range(0, n, _CHUNK):
        r1 = min(n, r0 + _CHUNK)
        x = _uniform(rng, (r1 - r0, dim)) * 0.05
        for j in range(rank):                       # the low-rank map as elementwise products, not a BLAS call
            x = x + latent[r0:r1, j:j + 1] * basis[j]
        out[r0:r1] = x / (1.0 + np.abs(x))
    return out


def make_queries(n: int, dim: int, seed: int, database: np.ndarray) -> np.ndarray:
    """[n, dim] float32: held-out points between consecutive trajectory rows of ``database`` plus small noise."""
    N, d = database.shape
    assert d == dim and N >= 2
    rng = np.random.Generator(np.random.PCG64(seed))
    i = rng.integers(0, N - 1, size=n)
    t = rng.random(n)[:, None]
    db = database.astype(np.float64)
    q = db[i] * (1.0 - t) + db[i + 1] * t + _uniform(rng, (n, dim)) * 0.02
    return q.astype(np.float32)


def make_singular_case(n_rows: int = 700, n: int = 8, dim: int = 512, seed: int = 5) -> Tuple[np.ndarray, np.ndarray, int, int]:
    """A database with one row duplicated exactly and queries whose row 0 sits on that row, so the two copies are its
    two nearest neighbours and the first column of ``A`` (neighbour 1 - neighbour 0) is exactly zero: the normal
    equations are singular and ``numpy.linalg.solve`` raises ``LinAlgError``.  Returns (database, queries, src, dst)."""
    db = make_database(n_rows, dim, seed)
    src, dst = n_rows // 3, (2 * n_rows) // 3
    db[dst] = db[src]
    q = make_queries(n, dim, seed + 1, db)
    q[0] = db[src]
    return db, q, src, dst


def sha256(a: np.ndarray) -> str:
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


# ------------------------------------------------------------------------------------------------------------------
# Restatement of the reference (fp32, same calls)
# ------------------------------------------------------------------------------------------------------------------
def knn_with_torch(feats: np.ndarray, feat_database: np.ndarray, K: int = 10) -> np.ndarray:
    """funcs/utils.py:100-116.  The reference's ``.cuda()`` calls are commented out: this runs on the host in fp32."""
    q = torch.from_numpy(feats)
    db = torch.from_numpy(feat_database)
    db_norm = (db ** 2).sum(-1)                                           # :104
    q_norm = (q ** 2).sum(-1)                                             # :107
    dist = q_norm.view(-1, 1) + db_norm.view(1, -1) - 2 * q @ db.t()      # :108-111
    return dist.topk(K, dim=1, largest=False).indices.cpu().numpy()       # :112, :116


def solve_lle_projection(feat: np.ndarray, feat_base: np.ndarray):
    """funcs/utils.py:121-157: min |feat - w.feat_base| s.t. sum(w) = 1, eliminated to (K-1) unknowns."""
    K, _ = feat_base.shape
    if K == 1:                                                            # :145-147
        return np.array([1]), feat_base[0]
    w = np.zeros(K)
    B = feat - feat_base[0]                                               # :150
    A = (feat_base[1:] - feat_base[0]).T                                  # :151  [ndim, K-1]
    At = A.T
    w[1:] = np.linalg.solve(At.dot(A), At.dot(B))                         # :153  fp32 LAPACK gesv
    w[0] = 1 - w[1:].sum()                                                # :154
    return w, w.dot(feat_base)                                            # :155  float64 result


def compute_lle_projection_all(feats: np.ndarray, feat_database: np.ndarray, ind: np.ndarray):
    """funcs/utils.py:171-179 (``nframe`` is recomputed from ``feats`` there, so it is not an argument here)."""
    n = feats.shape[0]
    feat_fuse = np.zeros_like(feats)
    w = np.zeros([n, ind.shape[1]])
    for i in range(n):
        w[i], feat_fuse[i] = solve_lle_projection(feats[i], feat_database[ind[i]])
    return w, feat_fuse


# ------------------------------------------------------------------------------------------------------------------
# float64 truths
# ------------------------------------------------------------------------------------------------------------------
def lle_truth(feats: np.ndarray, feat_database: np.ndarray, ind: np.ndarray):
    """Exact LLE (float64 normal equations) of the same fp32 inputs.  Returns (w [n,K], fuse [n,dim], cond [n]) in
    float64; ``cond`` is the 2-norm condition number of the Gram matrix (1 for K = 1)."""
    fb = feat_database[ind].astype(np.float64)                            # [n, K, dim]
    f = feats.astype(np.float64)
    n, K, _ = fb.shape
    if K == 1:
        return np.ones((n, 1)), fb[:, 0].copy(), np.ones(n)
    A = fb[:, 1:] - fb[:, :1]                                             # [n, K-1, dim] (exact: differences of fp32)
    B = f - fb[:, 0]
    G = np.einsum("nad,nbd->nab", A, A)
    r = np.einsum("nad,nd->na", A, B)
    x = np.linalg.solve(G, r[..., None])[..., 0]
    w = np.concatenate([1.0 - x.sum(1, keepdims=True), x], axis=1)
    fuse = np.einsum("nk,nkd->nd", w, fb)
    return w, fuse, np.linalg.cond(G)


def exact_sqdist(feats: np.ndarray, feat_database: np.ndarray, ind: np.ndarray) -> np.ndarray:
    """float64 |q_i - d_ind[i,j]|^2 for given indices [n, K]."""
    diff = feat_database[ind].astype(np.float64) - feats.astype(np.float64)[:, None, :]
    return (diff * diff).sum(-1)


def exact_topk(feats: np.ndarray, feat_database: np.ndarray, k: int, device: Optional[torch.device] = None,
               chunk: int = 16384) -> Tuple[np.ndarray, np.ndarray]:
    """The ``k`` smallest float64 squared distances per query and their rows (ascending; ties to the lower row), the
    database streamed in chunks so the [n, N] matrix is never held.  ``device`` only chooses where the float64 products
    run (the CPU by default)."""
    dev = torch.device("cpu") if device is None else torch.device(device)
    q = torch.from_numpy(feats).to(dev, torch.float64)
    qn = (q * q).sum(1, keepdim=True)
    best_d = torch.full((q.shape[0], 0), 0.0, dtype=torch.float64, device=dev)
    best_i = torch.zeros((q.shape[0], 0), dtype=torch.int64, device=dev)
    for r0 in range(0, feat_database.shape[0], chunk):
        d = torch.from_numpy(feat_database[r0:r0 + chunk]).to(dev, torch.float64)
        dist = (qn + (d * d).sum(1)[None, :] - 2.0 * (q @ d.t())).clamp_min(0.0)
        idx = torch.arange(r0, r0 + d.shape[0], device=dev).expand_as(dist)
        cd, ci = torch.cat([best_d, dist], 1), torch.cat([best_i, idx], 1)
        kk = min(k, cd.shape[1])
        # stable sort on distance after sorting by index: ties resolve to the lower row
        order = torch.sort(cd, dim=1, stable=True).indices[:, :kk]
        best_d, best_i = torch.gather(cd, 1, order), torch.gather(ci, 1, order)
    return best_d.cpu().numpy(), best_i.cpu().numpy()


def check_knn_band(ind: np.ndarray, feats: np.ndarray, feat_database: np.ndarray, k: int,
                   oracle_ind: Optional[np.ndarray] = None, device: Optional[torch.device] = None) -> float:
    """Assert that ``ind`` [n, k] is a correct fp32 KNN result.  fp32 ranking (any summation order) may order near-ties
    differently from exact arithmetic, so with tau_i = 2^-20 (|q_i|^2 + max_j |d_j|^2) and s_K the K-th smallest exact
    distance: every row closer than s_K - tau must be returned, none farther than s_K + tau may be, the rows are
    non-decreasing in exact distance up to tau, and on rows whose exact gaps (through the (K+1)-th) all exceed 2 tau the
    result equals ``oracle_ind``.  Returns the fraction of rows compared with the oracle."""
    n = feats.shape[0]
    assert ind.shape == (n, k) and ind.dtype == np.int64
    assert ((ind >= 0) & (ind < feat_database.shape[0])).all()
    assert all(len(set(r)) == k for r in ind.tolist()), "a row was returned twice"
    kk = min(k + 1, feat_database.shape[0])
    ex_d, ex_i = exact_topk(feats, feat_database, kk, device=device)
    dn_max = float((feat_database.astype(np.float64) ** 2).sum(1).max())
    tau = 2.0 ** -20 * ((feats.astype(np.float64) ** 2).sum(1) + dn_max)
    s_k = ex_d[:, k - 1]
    got = exact_sqdist(feats, feat_database, ind)
    assert (got <= (s_k + tau)[:, None]).all(), "a returned row is farther than s_K + tau"
    must = ex_d[:, :k] < (s_k - tau)[:, None]
    present = (ex_i[:, :k, None] == ind[:, None, :]).any(-1)
    assert (present | ~must).all(), "a row closer than s_K - tau is missing"
    assert (np.diff(got, axis=1) >= -tau[:, None]).all(), "not ascending in exact distance up to tau"
    if oracle_ind is None:
        return 0.0
    clear = (np.diff(ex_d, axis=1) > 2 * tau[:, None]).all(1) if kk > 1 else np.ones(n, bool)
    assert np.array_equal(ind[clear], oracle_ind[clear]), "differs from the fp32 oracle on well-separated rows"
    return float(clear.mean())


# ------------------------------------------------------------------------------------------------------------------
# The live reference (only where the reference checkout exists)
# ------------------------------------------------------------------------------------------------------------------
def reference_available() -> bool:
    return os.path.isfile(REF_FILE)


def reference_functions() -> dict:
    """KNN_with_torch, solve_LLE_projection and compute_LLE_projection_all_frame lifted out of funcs/utils.py with ``ast``
    and executed unchanged (the module itself imports librosa through ``audio_funcs``).  ``tqdm`` is bound to a
    pass-through so the LLE loop prints no progress bar; it does not touch the values."""
    import warnings
    with warnings.catch_warnings():                # the reference's docstrings contain "\s" escapes
        warnings.simplefilter("ignore", SyntaxWarning)
        tree = ast.parse(open(REF_FILE).read())
        wanted = ("KNN_with_torch", "solve_LLE_projection", "compute_LLE_projection_all_frame")
        funcs = [node for node in tree.body if isinstance(node, ast.FunctionDef) and node.name in wanted]
        assert sorted(f.name for f in funcs) == sorted(wanted)
        mod = ast.Module(body=funcs, type_ignores=[])
        ns: dict = {"np": np, "torch": torch, "solve": np.linalg.solve, "tqdm": lambda it, **kw: it}
        exec(compile(ast.fix_missing_locations(mod), REF_FILE, "exec"), ns)
    return {name: ns[name] for name in wanted}
