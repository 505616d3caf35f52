// C-ABI implementation of the APC manifold projection (see include/lspm.h; SURVEY.md 8f row N5).
//
// Reference: funcs/utils.py KNN_with_torch (:100-116) forms the full [n, N] fp32 distance matrix
// |q|^2 + |d|^2 - 2 q.d on the host and takes topk(K, largest=False); compute_LLE_projection_all_frame (:171-179) loops
// over the rows in Python, each one a (K-1)x(K-1) fp32 normal-equation solve (solve_LLE_projection, :121-157).
//
// Here:
//   * lspm_knn_kernel: a 128-query x 64-row fp32 distance tile per step (CUDA-core FMAs, dot products summed per 32-wide
//     slice of the feature dimension and then across slices), fused with a running per-query top-K kept in shared
//     memory, so the distance matrix never leaves the SM.  The grid is query tiles x database slices, sized to fill the
//     132 SMs once at two CTAs per SM; each CTA writes the K best (distance, row) pairs of its slice to the workspace.
//   * lspm_knn_merge_kernel: one warp per query merges the slices' lists.  Every list (in the CTAs and here) is ordered
//     by (distance, row), a total order, so the result does not depend on scheduling: ties go to the lower row.
//   * lspm_lle_kernel<EPL>: one warp per row gathers its K neighbours, forms A = [d_j - d_0], B = q - d_0 (exact in
//     fp64: differences of fp32 values), accumulates the Gram matrix A^T A and A^T B in fp64 (EPL entries of the upper
//     triangle per lane), solves by LU with partial pivoting in fp64, sets w0 = 1 - sum(w[1:]), and forms
//     fuse = w . d in fp64, rounded to fp32, and blend = q * (1 - p) + fuse * p in fp32 as the reference does.
// No kernel allocates; the database and its fp32 row norms are uploaded once by lspm_load_database.
#include <cuda_runtime.h>

#include <climits>
#include <cmath>

#include "../../include/lspm.h"
#include "capi.cuh"

using capi::align256;
using capi::DeviceGuard;

namespace {

struct Lspm;
constexpr auto fail = capi::fail<Lspm>;

constexpr int kMaxK = 32;        // neighbours: one warp lane per list entry
constexpr int kMaxDim = 1024;
constexpr int kTQ = 128;         // queries per distance tile
constexpr int kTN = 64;          // database rows per distance tile
constexpr int kTK = 32;          // feature columns per shared-memory stage (dim is a multiple of 32)
constexpr int kKnnThreads = 256; // 16 x 16 threads, 8 queries x 4 rows each
constexpr int kSMs = 132;        // H100 SXM
constexpr int kKnnCtasPerSM = 2;
constexpr int kLleWarps = 4;
constexpr unsigned kFull = 0xffffffffu;

struct KnnSmem {
  float qs[kTK][kTQ + 4];        // query stage, feature-major
  float ds[kTK][kTN + 4];        // database stage, feature-major
  float dist[kTQ][kTN + 1];      // the tile's distances
  float topd[kTQ][kMaxK];        // running top-K per query, ascending by (distance, row)
  int topi[kTQ][kMaxK];
};

__device__ __forceinline__ bool before(float ad, int ai, float bd, int bi) { return ad < bd || (ad == bd && ai < bi); }

// Insert this lane's candidate (if `want`) into the warp's sorted list (lane j holds entry j; entries >= k are ignored).
// Candidates are taken one at a time in lane order; each is placed by counting the entries before it, so the list
// stays sorted and a candidate that no longer beats entry k-1 is dropped.
__device__ __forceinline__ void warp_insert(bool want, float cd, int ci, float& ld, int& li, int k, int lane) {
  unsigned m = __ballot_sync(kFull, want);
  while (m) {
    const int src = __ffs(m) - 1;
    m &= m - 1;
    const float xd = __shfl_sync(kFull, cd, src);
    const int xi = __shfl_sync(kFull, ci, src);
    const int pos = __popc(__ballot_sync(kFull, lane < k && before(ld, li, xd, xi)));
    const float ud = __shfl_up_sync(kFull, ld, 1);
    const int ui = __shfl_up_sync(kFull, li, 1);
    if (pos < k) {
      if (lane == pos) { ld = xd; li = xi; }
      else if (lane > pos) { ld = ud; li = ui; }
    }
  }
}

// fp32 |x|^2 per row, one warp per row (lane-strided partial sums, then a butterfly).
__global__ void __launch_bounds__(256) lspm_norms_kernel(const float* __restrict__ x, int rows, int dim,
                                                         float* __restrict__ out) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* r = x + static_cast<size_t>(row) * dim;
  float s = 0.f;
  for (int d = lane; d < dim; d += 32) s = fmaf(r[d], r[d], s);
#pragma unroll
  for (int off = 16; off; off >>= 1) s += __shfl_xor_sync(kFull, s, off);
  if (lane == 0) out[row] = s;
}

__global__ void __launch_bounds__(kKnnThreads, kKnnCtasPerSM)
lspm_knn_kernel(const float* __restrict__ q, const float* __restrict__ qn, int n, const float* __restrict__ db,
                const float* __restrict__ dn, int n_rows, int dim, int k, int rows_per_slice, int slices,
                float* __restrict__ cand_d, int* __restrict__ cand_i) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  KnnSmem& sm = *reinterpret_cast<KnnSmem*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tx = tid & 15, ty = tid >> 4;
  const int q0 = blockIdx.x * kTQ, s = blockIdx.y;
  const int r_begin = s * rows_per_slice, r_end = min(n_rows, r_begin + rows_per_slice);
  for (int i = tid; i < kTQ * kMaxK; i += kKnnThreads) {
    sm.topd[i / kMaxK][i % kMaxK] = INFINITY;
    sm.topi[i / kMaxK][i % kMaxK] = INT_MAX;
  }
  float qnorm[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) qnorm[i] = (q0 + ty * 8 + i < n) ? qn[q0 + ty * 8 + i] : 0.f;

  for (int r0 = r_begin; r0 < r_end; r0 += kTN) {
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int k0 = 0; k0 < dim; k0 += kTK) {
#pragma unroll
      for (int e = tid; e < kTQ * kTK / 4; e += kKnnThreads) {
        const int row = e >> 3, c = (e & 7) * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (q0 + row < n) v = __ldg(reinterpret_cast<const float4*>(q + static_cast<size_t>(q0 + row) * dim + k0 + c));
        sm.qs[c][row] = v.x; sm.qs[c + 1][row] = v.y; sm.qs[c + 2][row] = v.z; sm.qs[c + 3][row] = v.w;
      }
#pragma unroll
      for (int e = tid; e < kTN * kTK / 4; e += kKnnThreads) {
        const int row = e >> 3, c = (e & 7) * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (r0 + row < r_end) v = __ldg(reinterpret_cast<const float4*>(db + static_cast<size_t>(r0 + row) * dim + k0 + c));
        sm.ds[c][row] = v.x; sm.ds[c + 1][row] = v.y; sm.ds[c + 2][row] = v.z; sm.ds[c + 3][row] = v.w;
      }
      __syncthreads();
      float part[8][4];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) part[i][j] = 0.f;
#pragma unroll
      for (int kk = 0; kk < kTK; ++kk) {
        const float4 a0 = *reinterpret_cast<const float4*>(&sm.qs[kk][ty * 8]);
        const float4 a1 = *reinterpret_cast<const float4*>(&sm.qs[kk][ty * 8 + 4]);
        const float4 b = *reinterpret_cast<const float4*>(&sm.ds[kk][tx * 4]);
        const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) part[i][j] = fmaf(a[i], bb[j], part[i][j]);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] += part[i][j];
      __syncthreads();
    }
    // (|q|^2 + |d|^2) - 2 q.d, rounded as the reference's fp32 expression is (2 q.d is exact)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int row = r0 + tx * 4 + j;
      const float dnorm = row < r_end ? dn[row] : 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i)
        sm.dist[ty * 8 + i][tx * 4 + j] = __fsub_rn(__fadd_rn(qnorm[i], dnorm), 2.f * acc[i][j]);
    }
    __syncthreads();
    // each warp folds the tile into the lists of its 16 queries; the next tile's first barrier orders these reads
    // before dist is written again
    for (int qq = 0; qq < kTQ / 8; ++qq) {
      const int qi = warp * (kTQ / 8) + qq;
      if (q0 + qi >= n) break;
      float ld = sm.topd[qi][lane];
      int li = sm.topi[qi][lane];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int c = lane + 32 * h;
        const float cd = sm.dist[qi][c];
        const int ci = r0 + c;
        const float td = __shfl_sync(kFull, ld, k - 1);
        const int ti = __shfl_sync(kFull, li, k - 1);
        warp_insert(ci < r_end && before(cd, ci, td, ti), cd, ci, ld, li, k, lane);
      }
      sm.topd[qi][lane] = ld;
      sm.topi[qi][lane] = li;
    }
  }
  for (int qq = 0; qq < kTQ / 8; ++qq) {
    const int qi = warp * (kTQ / 8) + qq;
    if (q0 + qi >= n) break;
    if (lane < k) {
      const size_t o = (static_cast<size_t>(q0 + qi) * slices + s) * k + lane;
      cand_d[o] = sm.topd[qi][lane];
      cand_i[o] = sm.topi[qi][lane];
    }
  }
}

__global__ void __launch_bounds__(256) lspm_knn_merge_kernel(const float* __restrict__ cand_d, const int* __restrict__ cand_i,
                                                             int n, int slices, int k, int64_t* __restrict__ out_ind,
                                                             float* __restrict__ out_dist) {
  const int qrow = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (qrow >= n) return;
  float ld = INFINITY;
  int li = INT_MAX;
  for (int s = 0; s < slices; ++s) {
    const size_t o = (static_cast<size_t>(qrow) * slices + s) * k + lane;
    const float cd = lane < k ? cand_d[o] : INFINITY;
    const int ci = lane < k ? cand_i[o] : INT_MAX;
    const float td = __shfl_sync(kFull, ld, k - 1);
    const int ti = __shfl_sync(kFull, li, k - 1);
    warp_insert(lane < k && before(cd, ci, td, ti), cd, ci, ld, li, k, lane);
  }
  if (lane < k) {
    out_ind[static_cast<size_t>(qrow) * k + lane] = li;
    if (out_dist) out_dist[static_cast<size_t>(qrow) * k + lane] = ld;
  }
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(kFull, v, off);
  return v;
}

// EPL: Gram entries per lane; the upper triangle of [A | B]^T [A | B] has k (k + 1) / 2 entries <= 32 * EPL.
template <int EPL>
__global__ void __launch_bounds__(kLleWarps * 32) lspm_lle_kernel(const float* __restrict__ feats, int n,
                                                                  const float* __restrict__ db, int64_t n_rows, int dim,
                                                                  const int64_t* __restrict__ ind, int k, float p,
                                                                  float one_minus_p, double* __restrict__ out_w,
                                                                  float* __restrict__ out_fuse, float* __restrict__ out_blend,
                                                                  int* __restrict__ out_status) {
  __shared__ double stage[kLleWarps][32][33];   // per warp: 32 feature rows x [A | B], then the augmented Gram matrix
  __shared__ int nbr[kLleWarps][kMaxK];
  __shared__ double wsh[kLleWarps][kMaxK];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * kLleWarps + warp;
  if (row >= n) return;                         // warps are independent: no block-wide barrier below
  const float* f = feats + static_cast<size_t>(row) * dim;
  const int64_t id = lane < k ? ind[static_cast<size_t>(row) * k + lane] : 0;
  int status = __any_sync(kFull, id < 0 || id >= n_rows) ? 2 : 0;
  double (*st)[33] = stage[warp];
  double wl = 0.0;                              // lane j: w[j]
  if (status == 0) {
    nbr[warp][lane] = static_cast<int>(id);
    __syncwarp();
    if (k == 1) {
      wl = 1.0;                                 // funcs/utils.py:145-147
    } else {
      const int m = k - 1, ncol = k;            // columns 0..m-1: A, column m: B
      const int total = ncol * (ncol + 1) / 2;
      int ab[EPL];
      double acc[EPL];
#pragma unroll
      for (int j = 0; j < EPL; ++j) {
        int e = lane + 32 * j, a = 0;
        if (e < total)
          while (e >= ncol - a) { e -= ncol - a; ++a; }
        ab[j] = a | ((a + e) << 8);
        acc[j] = 0.0;
      }
      const float* d0 = db + static_cast<size_t>(nbr[warp][0]) * dim;
      for (int c0 = 0; c0 < dim; c0 += 32) {
        const int c = c0 + lane;
        const double base = static_cast<double>(d0[c]);
        for (int j = 0; j < m; ++j) st[lane][j] = static_cast<double>(db[static_cast<size_t>(nbr[warp][j + 1]) * dim + c]) - base;
        st[lane][m] = static_cast<double>(f[c]) - base;
        __syncwarp();
#pragma unroll
        for (int j = 0; j < EPL; ++j) {
          if (lane + 32 * j < total) {
            const int a = ab[j] & 0xff, b = ab[j] >> 8;
            double s = acc[j];
#pragma unroll 8
            for (int r = 0; r < 32; ++r) s = fma(st[r][a], st[r][b], s);
            acc[j] = s;
          }
        }
        __syncwarp();
      }
      // augmented system G x = r: st[a][b] = (A^T A)[a][b], st[a][m] = (A^T B)[a]
#pragma unroll
      for (int j = 0; j < EPL; ++j) {
        if (lane + 32 * j < total) {
          const int a = ab[j] & 0xff, b = ab[j] >> 8;
          st[a][b] = acc[j];
          if (b < m) st[b][a] = acc[j];
        }
      }
      __syncwarp();
      // LU with partial pivoting (largest |pivot|, first on ties); lane c owns column c of the augmented matrix
      for (int kc = 0; kc < m; ++kc) {
        double v = (lane >= kc && lane < m) ? fabs(st[lane][kc]) : -1.0;
        int pr = lane;
#pragma unroll
        for (int off = 16; off; off >>= 1) {
          const double ov = __shfl_xor_sync(kFull, v, off);
          const int op = __shfl_xor_sync(kFull, pr, off);
          if (ov > v || (ov == v && op < pr)) { v = ov; pr = op; }
        }
        if (v == 0.0) { status = 1; break; }    // an exactly zero pivot: numpy.linalg.solve raises LinAlgError
        if (pr != kc && lane <= m) {
          const double t = st[kc][lane];
          st[kc][lane] = st[pr][lane];
          st[pr][lane] = t;
        }
        __syncwarp();
        const double piv = st[kc][kc];
        if (lane > kc && lane <= m)
          for (int r = kc + 1; r < m; ++r) st[r][lane] = fma(-(st[r][kc] / piv), st[kc][lane], st[r][lane]);
        __syncwarp();
      }
      if (status == 0) {
        double x = 0.0;                         // lane c: x[c]
        for (int r = m - 1; r >= 0; --r) {
          const double t = warp_sum((lane > r && lane < m) ? st[r][lane] * x : 0.0);
          const double xr = (st[r][m] - t) / st[r][r];
          if (lane == r) x = xr;
        }
        const double up = __shfl_up_sync(kFull, x, 1);
        wl = (lane >= 1 && lane <= m) ? up : 0.0;
        const double w0 = 1.0 - warp_sum(wl);   // funcs/utils.py:154
        if (lane == 0) wl = w0;
      }
    }
  }
  if (status != 0) {
    const float fnan = __int_as_float(0x7fc00000);
    if (out_w && lane < k) out_w[static_cast<size_t>(row) * k + lane] = __longlong_as_double(0x7ff8000000000000LL);
    for (int c = lane; c < dim; c += 32) {
      if (out_fuse) out_fuse[static_cast<size_t>(row) * dim + c] = fnan;
      if (out_blend) out_blend[static_cast<size_t>(row) * dim + c] = fnan;
    }
    if (out_status && lane == 0) out_status[row] = status;
    return;
  }
  if (out_w && lane < k) out_w[static_cast<size_t>(row) * k + lane] = wl;
  if (out_status && lane == 0) out_status[row] = 0;
  if (!out_fuse && !out_blend) return;
  wsh[warp][lane] = wl;
  __syncwarp();
  for (int c = lane; c < dim; c += 32) {
    double s = 0.0;
    for (int j = 0; j < k; ++j) s = fma(wsh[warp][j], static_cast<double>(db[static_cast<size_t>(nbr[warp][j]) * dim + c]), s);
    const float fuse = static_cast<float>(s);   // funcs/utils.py:155, stored into the float32 feat_fuse (:177)
    if (out_fuse) out_fuse[static_cast<size_t>(row) * dim + c] = fuse;
    if (out_blend) out_blend[static_cast<size_t>(row) * dim + c] = __fadd_rn(__fmul_rn(f[c], one_minus_p), __fmul_rn(fuse, p));
  }
}

int ceil_div(int a, int b) { return (a + b - 1) / b; }

// Database slices per query tile: fill kSMs x kKnnCtasPerSM CTAs once.  Depends on n only, so the workspace size does
// not depend on the database; the launch uses min(this, number of 64-row tiles).
int max_slices(int n) { return ceil_div(kSMs * kKnnCtasPerSM, ceil_div(n, kTQ)); }

size_t workspace_bytes(int n, int k) {
  const size_t cand = static_cast<size_t>(n) * max_slices(n) * k;
  return align256(sizeof(float) * n) + align256(sizeof(float) * cand) + align256(sizeof(int) * cand);
}

}  // namespace

struct lspm_ctx {
  int dim = 0;
  int device = -1;
  int64_t n_rows = 0;
  float* d_db = nullptr;
  float* d_norm = nullptr;
};

extern "C" {

const char* lspm_last_error(void) { return capi::last_error<Lspm>().c_str(); }

int lspm_create(lspm_handle* out, int dim, int device) {
  if (!out) return fail(LSPG_EINVAL, "null argument");
  *out = nullptr;
  if (dim < 32 || dim > kMaxDim || dim % 32) return fail(LSPG_EINVAL, "dim must be a multiple of 32 in [32, %d] (got %d)", kMaxDim, dim);
  cudaDeviceProp prop;
  if (int rc = capi::check_device<Lspm>(device, &prop)) return rc;
  if (device >= 0) {
    DeviceGuard g(device);
    CUDA_TRY(cudaFuncSetAttribute(lspm_knn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(sizeof(KnnSmem))));
  }
  lspm_ctx* h = new lspm_ctx;
  h->dim = dim;
  h->device = device;
  *out = h;
  return LSPG_OK;
}

int lspm_load_database(lspm_handle h, const float* host_db, int64_t n_rows) {
  if (!h || !host_db) return fail(LSPG_EINVAL, "null argument");
  if (n_rows < 1 || n_rows >= (static_cast<int64_t>(1) << 31)) return fail(LSPG_EINVAL, "n_rows must be in [1, 2^31) (got %lld)", static_cast<long long>(n_rows));
  if (int rc = capi::require_device<Lspm>(h->device, "lspm_load_database")) return rc;
  DeviceGuard g(h->device);
  if (n_rows != h->n_rows) {
    if (h->d_db) cudaFree(h->d_db);
    if (h->d_norm) cudaFree(h->d_norm);
    h->d_db = nullptr; h->d_norm = nullptr; h->n_rows = 0;
    CUDA_TRY(cudaMalloc(&h->d_db, sizeof(float) * static_cast<size_t>(n_rows) * h->dim));
    CUDA_TRY(cudaMalloc(&h->d_norm, sizeof(float) * static_cast<size_t>(n_rows)));
  }
  h->n_rows = 0;                                // not usable until the copy and the norms are complete
  CUDA_TRY(cudaMemcpy(h->d_db, host_db, sizeof(float) * static_cast<size_t>(n_rows) * h->dim, cudaMemcpyHostToDevice));
  lspm_norms_kernel<<<ceil_div(static_cast<int>(n_rows), 8), 256>>>(h->d_db, static_cast<int>(n_rows), h->dim, h->d_norm);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaStreamSynchronize(0));
  h->n_rows = n_rows;
  return LSPG_OK;
}

int lspm_workspace_bytes(lspm_handle h, int n, int k, size_t* out) {
  if (!h || !out) return fail(LSPG_EINVAL, "null argument");
  if (n < 1) return fail(LSPG_EINVAL, "n must be >= 1 (got %d)", n);
  if (k < 1 || k > kMaxK) return fail(LSPG_EINVAL, "k must be in [1, %d] (got %d)", kMaxK, k);
  *out = workspace_bytes(n, k);
  return LSPG_OK;
}

int lspm_knn(lspm_handle h, const float* feats, int n, int k, int64_t* out_ind, float* out_dist_or_null, void* ws,
             size_t ws_bytes, void* stream) {
  if (!h) return fail(LSPG_EINVAL, "null handle");
  if (n < 1) return fail(LSPG_EINVAL, "n must be >= 1 (got %d)", n);
  if (k < 1 || k > kMaxK) return fail(LSPG_EINVAL, "k must be in [1, %d] (got %d)", kMaxK, k);
  if (h->n_rows > 0 && k > h->n_rows) return fail(LSPG_EINVAL, "k (%d) exceeds the %lld database rows", k, static_cast<long long>(h->n_rows));
  if (!feats || !out_ind || !ws) return fail(LSPG_EINVAL, "null buffer");
  if (reinterpret_cast<uintptr_t>(feats) % 16) return fail(LSPG_EINVAL, "feats must be 16-byte aligned");
  const size_t need = workspace_bytes(n, k);
  if (ws_bytes < need) return fail(LSPG_EINVAL, "workspace of %zu bytes is smaller than the %zu needed", ws_bytes, need);
  if (int rc = capi::require_device<Lspm>(h->device, "lspm_knn")) return rc;
  if (h->n_rows == 0) return fail(LSPG_ESTATE, "lspm_load_database has not been called");
  DeviceGuard g(h->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int n_rows = static_cast<int>(h->n_rows);
  const int tiles = ceil_div(n_rows, kTN);
  int slices = max_slices(n) < tiles ? max_slices(n) : tiles;
  const int rows_per_slice = ceil_div(tiles, slices) * kTN;
  slices = ceil_div(n_rows, rows_per_slice);
  char* w = static_cast<char*>(ws);
  float* qn = reinterpret_cast<float*>(w);
  float* cand_d = reinterpret_cast<float*>(w + align256(sizeof(float) * n));
  const size_t cand = static_cast<size_t>(n) * max_slices(n) * k;
  int* cand_i = reinterpret_cast<int*>(w + align256(sizeof(float) * n) + align256(sizeof(float) * cand));
  lspm_norms_kernel<<<ceil_div(n, 8), 256, 0, st>>>(feats, n, h->dim, qn);
  lspm_knn_kernel<<<dim3(ceil_div(n, kTQ), slices), kKnnThreads, sizeof(KnnSmem), st>>>(
      feats, qn, n, h->d_db, h->d_norm, n_rows, h->dim, k, rows_per_slice, slices, cand_d, cand_i);
  lspm_knn_merge_kernel<<<ceil_div(n, 8), 256, 0, st>>>(cand_d, cand_i, n, slices, k, out_ind, out_dist_or_null);
  CUDA_TRY(cudaGetLastError());
  return LSPG_OK;
}

int lspm_project(lspm_handle h, const float* feats, int n, const int64_t* ind, int k, float percent, double* out_w,
                 float* out_fuse, float* out_blend, int* out_status, void* stream) {
  if (!h) return fail(LSPG_EINVAL, "null handle");
  if (n < 1) return fail(LSPG_EINVAL, "n must be >= 1 (got %d)", n);
  if (k < 1 || k > kMaxK) return fail(LSPG_EINVAL, "k must be in [1, %d] (got %d)", kMaxK, k);
  if (!feats || !ind) return fail(LSPG_EINVAL, "null buffer");
  if (int rc = capi::require_device<Lspm>(h->device, "lspm_project")) return rc;
  if (h->n_rows == 0) return fail(LSPG_ESTATE, "lspm_load_database has not been called");
  DeviceGuard g(h->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // demo.py:200 multiplies the float32 features by the Python float (1 - LLE_percent): that product is formed in
  // double and rounded to float32 once
  const float omp = static_cast<float>(1.0 - static_cast<double>(percent));
  const dim3 grid(ceil_div(n, kLleWarps)), block(kLleWarps * 32);
  const int entries = k * (k + 1) / 2;
  if (entries <= 64)
    lspm_lle_kernel<2><<<grid, block, 0, st>>>(feats, n, h->d_db, h->n_rows, h->dim, ind, k, percent, omp, out_w, out_fuse, out_blend, out_status);
  else if (entries <= 224)
    lspm_lle_kernel<7><<<grid, block, 0, st>>>(feats, n, h->d_db, h->n_rows, h->dim, ind, k, percent, omp, out_w, out_fuse, out_blend, out_status);
  else
    lspm_lle_kernel<17><<<grid, block, 0, st>>>(feats, n, h->d_db, h->n_rows, h->dim, ind, k, percent, omp, out_w, out_fuse, out_blend, out_status);
  CUDA_TRY(cudaGetLastError());
  return LSPG_OK;
}

int lspm_destroy(lspm_handle h) {
  if (!h) return LSPG_OK;
  if (h->device >= 0) {
    DeviceGuard g(h->device);
    if (h->d_db) cudaFree(h->d_db);
    if (h->d_norm) cudaFree(h->d_norm);
  }
  delete h;
  return LSPG_OK;
}

}  // extern "C"
