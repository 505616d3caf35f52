/*
 * lspm.h - C ABI of the H100-native APC manifold projection (LiveSpeechPortraits, SURVEY.md 8f row N5).
 *
 * What it replaces: stage 2 of demo.py (:196-200, predict.py:180-185) - funcs/utils.py KNN_with_torch (:100-116), an
 * fp32 GEMM of every APC feature row against the identity's feature base followed by topk, which runs on the HOST even
 * with --device cuda (its .cuda() calls are commented out), and compute_LLE_projection_all_frame (:171-179), a Python
 * loop of one (K-1)x(K-1) numpy.linalg.solve per row.  Here: one fused distance + top-K kernel (the [n, N] distance
 * matrix never reaches memory), one merge kernel and one LLE kernel that solves every row in fp64.
 *
 * Conventions as in lspg.h / lsph.h: plain C types, 0 or a negative LSPG_E* code, message in lspm_last_error(); sm_90
 * only, no CPU path.  All pointers except host_db are DEVICE pointers; every call after lspm_load_database is
 * asynchronous on `stream` and allocates nothing.  The Python binding is livespeechportraits_b200/manifold.py.
 */
#ifndef LSPM_H_
#define LSPM_H_

#include <stddef.h>
#include <stdint.h>

#include "lspg.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct lspm_ctx* lspm_handle;

/* dim: feature width (APC_hidden_size, 512 shipped), a multiple of 32 and at most 1024.  device == -1: host-only handle
 * (argument checking only; lspm_load_database / lspm_knn / lspm_project return LSPG_ENODEV). */
int lspm_create(lspm_handle* out, int dim, int device);

/* The identity's APC_feature_base.npy: host fp32 [n_rows, dim], 1 <= n_rows < 2^31.  Synchronous: copies to a
 * library-owned device buffer and computes the fp32 row norms |d|^2 there.  A second call replaces the database. */
int lspm_load_database(lspm_handle h, const float* host_db, int64_t n_rows);

/* Bytes of caller-owned device workspace lspm_knn needs for n query rows and k neighbours (independent of n_rows). */
int lspm_workspace_bytes(lspm_handle h, int n, int k, size_t* out);

/* KNN_with_torch: feats [n, dim] fp32 (16-byte aligned), 1 <= k <= min(32, n_rows).  out_ind [n, k] int64: per row the
 * k database rows of smallest  |q|^2 + |d|^2 - 2 q.d  (fp32, the reference's formula), ascending, ties to the lower
 * row.  out_dist_or_null [n, k] fp32: those distances. */
int lspm_knn(lspm_handle h, const float* feats, int n, int k, int64_t* out_ind, float* out_dist_or_null, void* ws,
             size_t ws_bytes, void* stream);

/* compute_LLE_projection_all_frame + the blend of demo.py:200, given ind [n, k] int64 (1 <= k <= 32):
 *   out_w     [n, k] fp64   the LLE weights (sum to 1; w = 1 for k = 1)
 *   out_fuse  [n, dim] fp32 w . database[ind[i]]
 *   out_blend [n, dim] fp32 feats * (1 - percent) + fuse * percent, in fp32 as the reference computes it
 *   out_status [n] int      0 ok, 1 singular (an exactly zero pivot - the reference raises LinAlgError),
 *                           2 an index outside [0, n_rows) (nothing is read through it)
 * Any output may be NULL.  Rows with a non-zero status get NaN in w, fuse and blend. */
int lspm_project(lspm_handle h, const float* feats, int n, const int64_t* ind, int k, float percent, double* out_w,
                 float* out_fuse, float* out_blend, int* out_status, void* stream);

int lspm_destroy(lspm_handle h);
const char* lspm_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* LSPM_H_ */
