// C-ABI implementation of the recurrent audio networks (see include/lspr.h): the APC encoder's GRU stack
// (models/networks.py:20-69) and Audio2Mouth's downsample MLP, 3-layer LSTM and fc MLP (models/audio2feature.py:32-69,
// driven by models/audio2feature_model.py:117-154).
//
// A recurrent layer is split in two:
//   * the input projection X W_ih^T + b of all T steps is one fp32 GEMM (gemm_nt_kernel, csrc/gemm_nt.cuh), with
//     b_ih + b_hh folded for every gate except the GRU's n gate, whose b_hn sits inside r * (W_hn h + b_hn);
//   * the recurrence is ONE persistent launch of one thread-block cluster of CL CTAs.  CTA c owns hidden units
//     [c H/CL, (c+1) H/CL): it keeps those units' W_hh rows of every gate in shared memory (fp32), forms their gates from
//     its own copy of h_{t-1}, applies the cell (the LSTM's c stays in a register), stores its slice of h_t into the
//     other buffer of every CTA's double-buffered h (st.shared::cluster), passes one cluster barrier (release/acquire)
//     and writes the slice to the layer output.  The double buffer makes one barrier per step enough: a CTA writes buffer
//     (t+1)&1 of its peers only after the barrier that ends step t - 1, which every peer passed after its last read of it.
//   * Shapes: the GRU (H = 512) runs 16 CTAs x 96 rows (192 KB of W_hh per CTA, a non-portable cluster size); when no
//     16-CTA cluster fits on the device it runs 8 CTAs x 192 rows, 96 of them in shared memory and 96 read from L2 every
//     step.  The LSTM (H = 256) runs 8 CTAs x 128 rows (128 KB).
// Every dot product is a per-lane fmaf chain followed by a fixed xor butterfly, expf/tanhf are the accurate ones and there
// are no atomics: repeated runs are bit-identical.
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/lspr.h"
#include "capi.cuh"
#include "gemm_nt.cuh"

namespace cg = cooperative_groups;
using capi::DeviceGuard;

namespace {

struct Lspr;
constexpr auto fail = capi::fail<Lspr>;

constexpr int kNW = 16;            // warps per CTA of the recurrence
constexpr int kApcH = 512;         // APC hidden size the GRU kernels are built for
constexpr int kLstmH = 256;        // models/audio2feature.py:40
constexpr int kFcW = 512;          // models/audio2feature.py:46-52
constexpr int kMaxApcLayers = 8;
constexpr int kMaxOut = 4096;

struct RecParams {
  const float* xproj;   // [T][G*H]: input projection + folded biases, gate rows interleaved by unit (row u*G + g)
  const float* w_hh;    // [G*H][H], same row order: CTA c's rows are the block [c*G*H/CL, (c+1)*G*H/CL)
  const float* b_hn;    // [H] (GRU) or null
  const float* resid;   // [T][H] added to the output (APC residual), or null
  float* out;           // [T][H]
  float* state;         // [2][H]: h (and the LSTM's c) before step 0, replaced by their values after step T-1; or null (zeros)
  int T;
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

template <int G, int H, int CL, int RS>
constexpr size_t rnn_smem_bytes() {
  return sizeof(float) * (static_cast<size_t>(RS) * H + 2 * H + G * (H / CL));
}

// G gates (3: GRU r, z, n; 4: LSTM i, f, g, o), H hidden units, CL CTAs, RS of the CTA's G*H/CL rows in shared memory.
// Warp w computes the CTA-local rows w, w + kNW, ...; rows below RS come from shared memory, the rest from global (L2).
template <int G, int H, int CL, int RS>
__global__ void __launch_bounds__(kNW * 32, 1) rnn_layer_kernel(const RecParams p) {
  constexpr int U = H / CL;          // hidden units per CTA
  constexpr int R = G * U;           // W_hh rows per CTA
  constexpr int RW = R / kNW;        // rows per warp
  constexpr int RSW = RS / kNW;      // of them in shared memory
  constexpr int V = H / 128;         // float4 per lane per row
  static_assert(R % kNW == 0 && RS % kNW == 0 && RS <= R && H % 128 == 0 && U <= kNW * 32, "bad recurrence shape");

  extern __shared__ __align__(16) float smem[];
  float* w_s = smem;                 // [RS][H]: local rows 0 .. RS-1
  float* h_s = smem + RS * H;        // [2][H]: h_{t-1} (buffer t&1) and h_t (the other)
  float* g_s = h_s + 2 * H;          // [R]: W_hh h_{t-1} of the local rows

  cg::cluster_group cluster = cg::this_cluster();
  const int c = static_cast<int>(cluster.block_rank());
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* w_cta = p.w_hh + static_cast<size_t>(c) * R * H;

  for (int i = tid; i < RS * H / 4; i += kNW * 32)
    reinterpret_cast<float4*>(w_s)[i] = __ldg(reinterpret_cast<const float4*>(w_cta) + i);
  for (int i = tid; i < 2 * H; i += kNW * 32) h_s[i] = (p.state && i < H) ? p.state[i] : 0.f;   // h_0 = 0 or the saved h
  const int u = c * U + tid;                                            // the unit this thread updates (tid < U)
  float cst = (G == 4 && p.state && tid < U) ? p.state[H + u] : 0.f;    // c_0 likewise
  float hlast = 0.f;
  float bhn = 0.f;
  float xg[G];
  if (tid < U) {
    if constexpr (G == 3) bhn = __ldg(p.b_hn + u);
    if (p.T > 0) {
#pragma unroll
      for (int g = 0; g < G; ++g) xg[g] = __ldg(p.xproj + static_cast<size_t>(u) * G + g);
    }
  }
  cluster.sync();                    // every CTA has started and zeroed its h before any peer stores into it

  int cur = 0;
  for (int t = 0; t < p.T; ++t) {
    float4 hv[V];
#pragma unroll
    for (int v = 0; v < V; ++v) hv[v] = reinterpret_cast<const float4*>(h_s + cur * H)[lane + 32 * v];
#pragma unroll
    for (int rr = 0; rr < RW; ++rr) {
      const int lr = warp + kNW * rr;
      float acc = 0.f;
#pragma unroll
      for (int v = 0; v < V; ++v) {
        const float4 w = rr < RSW ? reinterpret_cast<const float4*>(w_s + static_cast<size_t>(lr) * H)[lane + 32 * v]
                                  : __ldg(reinterpret_cast<const float4*>(w_cta + static_cast<size_t>(lr) * H) + lane + 32 * v);
        acc = fmaf(w.x, hv[v].x, acc);
        acc = fmaf(w.y, hv[v].y, acc);
        acc = fmaf(w.z, hv[v].z, acc);
        acc = fmaf(w.w, hv[v].w, acc);
      }
      acc = warp_sum(acc);
      if (lane == 0) g_s[lr] = acc;
    }
    __syncthreads();
    if (tid < U) {
      const float hp = h_s[cur * H + u];
      const float* gh = g_s + tid * G;
      float hn;
      if constexpr (G == 3) {        // torch GRU: n = tanh(W_in x + b_in + r (W_hn h + b_hn)),  h' = (1 - z) n + z h
        const float r = sigmoidf_(xg[0] + gh[0]);
        const float z = sigmoidf_(xg[1] + gh[1]);
        const float n = tanhf(xg[2] + r * (gh[2] + bhn));
        hn = n + z * (hp - n);
      } else {                       // torch LSTM: c' = f c + i g,  h' = o tanh(c')
        const float ig = sigmoidf_(xg[0] + gh[0]);
        const float fg = sigmoidf_(xg[1] + gh[1]);
        const float gg = tanhf(xg[2] + gh[2]);
        const float og = sigmoidf_(xg[3] + gh[3]);
        cst = fg * cst + ig * gg;
        hn = og * tanhf(cst);
      }
#pragma unroll
      for (int r = 0; r < CL; ++r) cluster.map_shared_rank(h_s, r)[(cur ^ 1) * H + u] = hn;
      const size_t o = static_cast<size_t>(t) * H + u;
      p.out[o] = p.resid ? hn + p.resid[o] : hn;
      hlast = hn;
      if (t + 1 < p.T) {
#pragma unroll
        for (int g = 0; g < G; ++g) xg[g] = __ldg(p.xproj + (static_cast<size_t>(t + 1) * H + u) * G + g);
      }
    }
    cluster.sync();                  // h_t complete in every CTA
    cur ^= 1;
  }
  // Every CTA read the saved state before the first step's barrier, so the units' owners may now replace it.
  if (p.state && p.T > 0 && tid < U) {
    p.state[u] = hlast;
    if constexpr (G == 4) p.state[H + u] = cst;
  }
}

// The three recurrence shapes.
constexpr int kGruRows16 = 3 * kApcH / 16;     // 96 rows per CTA, all in shared memory
constexpr int kLstmRows8 = 4 * kLstmH / 8;     // 128
#define GRU16 rnn_layer_kernel<3, kApcH, 16, kGruRows16>
#define GRU8 rnn_layer_kernel<3, kApcH, 8, kGruRows16>
#define LSTM8 rnn_layer_kernel<4, kLstmH, 8, kLstmRows8>
constexpr size_t kGru16Smem = rnn_smem_bytes<3, kApcH, 16, kGruRows16>();
constexpr size_t kGru8Smem = rnn_smem_bytes<3, kApcH, 8, kGruRows16>();
constexpr size_t kLstm8Smem = rnn_smem_bytes<4, kLstmH, 8, kLstmRows8>();

size_t align_floats(size_t n) { return (n + 63) / 64 * 64; }

}  // namespace

struct lspr_ctx {
  lspr_config cfg{};
  int device = -1;
  int G = 0, H = 0, L = 0;
  std::vector<int> in_w;                       // input width of each recurrent layer
  bool weights_loaded = false;
  std::vector<std::vector<float>> packed;      // lspr_debug_packed order
  std::vector<float*> d_packed;                // device copies, same order
  float* d_ones = nullptr;
  size_t n_ones = 0;
  int max_clusters16 = 0, max_clusters8 = 0;   // cudaOccupancyMaxActiveClusters of the recurrence launches
};

namespace {

int launch_rnn(lspr_ctx* h, int cl, const RecParams& p, cudaStream_t st) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(cl);
  cfg.blockDim = dim3(kNW * 32);
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cl; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  if (h->G == 4) {
    cfg.dynamicSmemBytes = kLstm8Smem;
    CUDA_TRY(cudaLaunchKernelEx(&cfg, LSTM8, p));
  } else if (cl == 16) {
    cfg.dynamicSmemBytes = kGru16Smem;
    CUDA_TRY(cudaLaunchKernelEx(&cfg, GRU16, p));
  } else {
    cfg.dynamicSmemBytes = kGru8Smem;
    CUDA_TRY(cudaLaunchKernelEx(&cfg, GRU8, p));
  }
  return LSPG_OK;
}

template <typename K>
int max_clusters(K kernel, int cl, size_t smem, int* out) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(cl);
  cfg.blockDim = dim3(kNW * 32);
  cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cl; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  if (cl > 8) CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  *out = 0;
  if (cudaOccupancyMaxActiveClusters(out, kernel, &cfg) != cudaSuccess) {
    cudaGetLastError();              // "cannot be scheduled" comes back as an error on some drivers: treat it as 0
    *out = 0;
  }
  return LSPG_OK;
}

void gemm(const float* A, const float* W, const float* scale, const float* shift, float* C, int M, int N, int K, int leaky,
          cudaStream_t st) {
  gemm_nt_kernel<><<<dim3(N / 64, (M + 63) / 64), 256, 0, st>>>(A, W, scale, shift, C, M, N, K, leaky);
}

}  // namespace

extern "C" {

const char* lspr_last_error(void) { return capi::last_error<Lspr>().c_str(); }

int lspr_create(lspr_handle* out, const lspr_config* c, int device) {
  if (!out || !c) return fail(LSPG_EINVAL, "null argument");
  *out = nullptr;
  std::unique_ptr<lspr_ctx> h(new lspr_ctx);
  h->cfg = *c;
  h->device = device;
  if (c->kind == LSPR_APC) {
    if (c->hidden != kApcH) return fail(LSPG_EINVAL, "APC hidden_size must be %d (got %d)", kApcH, c->hidden);
    if (c->input_dim < 16 || c->input_dim % 16) return fail(LSPG_EINVAL, "APC mel_dim must be a positive multiple of 16 (got %d)", c->input_dim);
    if (c->num_layers < 1 || c->num_layers > kMaxApcLayers) return fail(LSPG_EINVAL, "APC num_layers must be in [1, %d] (got %d)", kMaxApcLayers, c->num_layers);
    h->G = 3; h->H = kApcH; h->L = c->num_layers;
    for (int l = 0; l < h->L; ++l) h->in_w.push_back(l == 0 ? c->input_dim : kApcH);
  } else if (c->kind == LSPR_MOUTH) {
    if (c->input_dim < 64 || c->input_dim % 64) return fail(LSPG_EINVAL, "APC_hidden_size must be a positive multiple of 64 (got %d)", c->input_dim);
    if (c->frame_future < 0) return fail(LSPG_EINVAL, "frame_future must be >= 0 (got %d)", c->frame_future);
    if (c->out_dim < 1 || c->out_dim > kMaxOut) return fail(LSPG_EINVAL, "out_dim must be in [1, %d] (got %d)", kMaxOut, c->out_dim);
    h->G = 4; h->H = kLstmH; h->L = 3;
    for (int l = 0; l < h->L; ++l) h->in_w.push_back(l == 0 ? c->input_dim : kLstmH);
  } else {
    return fail(LSPG_EINVAL, "kind must be LSPR_APC or LSPR_MOUTH (got %d)", c->kind);
  }
  cudaDeviceProp prop;
  if (int rc = capi::check_device<Lspr>(device, &prop)) return rc;
  if (device >= 0) {
    DeviceGuard g(device);
    int r;
    if (h->G == 3) {
      if ((r = max_clusters(GRU16, 16, kGru16Smem, &h->max_clusters16))) return r;
      if ((r = max_clusters(GRU8, 8, kGru8Smem, &h->max_clusters8))) return r;
    } else {
      if ((r = max_clusters(LSTM8, 8, kLstm8Smem, &h->max_clusters8))) return r;
    }
  }
  *out = h.release();
  return LSPG_OK;
}

int lspr_destroy(lspr_handle h) {
  if (!h) return LSPG_OK;
  if (h->device >= 0) {
    DeviceGuard g(h->device);
    for (float* p : h->d_packed) if (p) cudaFree(p);
    if (h->d_ones) cudaFree(h->d_ones);
  }
  delete h;
  return LSPG_OK;
}

int lspr_load_weights(lspr_handle h, const lspg_tensor* tensors, int n) {
  if (!h || (!tensors && n > 0)) return fail(LSPG_EINVAL, "null argument");
  const lspr_config& c = h->cfg;
  capi::WeightTable<Lspr> wt(tensors, n);
  if (int rc = wt.status()) return rc;
  const int G = h->G, H = h->H;
  std::vector<std::vector<float>> packed;
  // ---- recurrent layers: gate rows interleaved by unit, biases folded except the GRU's b_hn
  for (int l = 0; l < h->L; ++l) {
    const int In = h->in_w[l];
    const std::string p = c.kind == LSPR_APC ? "rnns." + std::to_string(l) + "." : "LSTM.";
    const std::string sfx = c.kind == LSPR_APC ? "_l0" : "_l" + std::to_string(l);
    const float* wih = wt.get(p + "weight_ih" + sfx, static_cast<size_t>(G) * H * In);
    const float* whh = wt.get(p + "weight_hh" + sfx, static_cast<size_t>(G) * H * H);
    const float* bih = wt.get(p + "bias_ih" + sfx, static_cast<size_t>(G) * H);
    const float* bhh = wt.get(p + "bias_hh" + sfx, static_cast<size_t>(G) * H);
    if (int rc = wt.status()) return rc;
    std::vector<float> w_ih(static_cast<size_t>(G) * H * In), b(static_cast<size_t>(G) * H), w_hh(static_cast<size_t>(G) * H * H);
    std::vector<float> b_hn(G == 3 ? H : 0);
    for (int u = 0; u < H; ++u)
      for (int g = 0; g < G; ++g) {
        const size_t src = static_cast<size_t>(g) * H + u, dst = static_cast<size_t>(u) * G + g;
        memcpy(&w_ih[dst * In], wih + src * In, sizeof(float) * In);
        memcpy(&w_hh[dst * H], whh + src * H, sizeof(float) * H);
        b[dst] = (G == 3 && g == 2) ? bih[src] : bih[src] + bhh[src];
        if (G == 3 && g == 2) b_hn[u] = bhh[src];
      }
    packed.push_back(std::move(w_ih));
    packed.push_back(std::move(b));
    packed.push_back(std::move(w_hh));
    packed.push_back(std::move(b_hn));
  }
  // ---- Audio2Mouth MLPs: Linear (+ eval BatchNorm1d folded into scale / shift)
  if (c.kind == LSPR_MOUTH) {
    const int D = c.input_dim;
    struct Stage { const char* lin; const char* bn; int n, k; };
    const Stage stages[5] = {{"downsample.0", "downsample.1", D, 2 * D}, {"downsample.3", nullptr, D, D},
                             {"fc.0", "fc.1", kFcW, kLstmH}, {"fc.3", "fc.4", kFcW, kFcW}, {"fc.6", nullptr, c.out_dim, kFcW}};
    for (const Stage& s : stages) {
      const std::string lin = s.lin;
      const float* w = wt.get(lin + ".weight", static_cast<size_t>(s.n) * s.k);
      const float* bias = wt.get(lin + ".bias", s.n);
      const float *bw = nullptr, *bb = nullptr, *bm = nullptr, *bv = nullptr;
      if (s.bn) {
        const std::string bn = s.bn;
        bw = wt.get(bn + ".weight", s.n); bb = wt.get(bn + ".bias", s.n);
        bm = wt.get(bn + ".running_mean", s.n); bv = wt.get(bn + ".running_var", s.n);
      }
      if (int rc = wt.status()) return rc;
      std::vector<float> scale(s.n, 1.0f), shift(bias, bias + s.n);
      if (s.bn)
        for (int j = 0; j < s.n; ++j) {
          const float sc = bw[j] / sqrtf(bv[j] + 1e-5f);      // BatchNorm1d eval, eps = torch default
          scale[j] = sc;
          shift[j] = (bias[j] - bm[j]) * sc + bb[j];
        }
      packed.emplace_back(w, w + static_cast<size_t>(s.n) * s.k);
      packed.push_back(std::move(scale));
      packed.push_back(std::move(shift));
    }
  }
  if (h->device >= 0) {
    DeviceGuard g(h->device);
    CUDA_TRY(cudaDeviceSynchronize());          // no launch still reads the arrays being replaced
    if (h->d_packed.size() != packed.size()) h->d_packed.assign(packed.size(), nullptr);
    for (size_t i = 0; i < packed.size(); ++i) {
      if (h->d_packed[i] && (h->packed.size() != packed.size() || h->packed[i].size() != packed[i].size())) {
        cudaFree(h->d_packed[i]);
        h->d_packed[i] = nullptr;
      }
      if (!h->d_packed[i] && !packed[i].empty()) CUDA_TRY(cudaMalloc(&h->d_packed[i], sizeof(float) * packed[i].size()));
      if (!packed[i].empty())
        CUDA_TRY(cudaMemcpy(h->d_packed[i], packed[i].data(), sizeof(float) * packed[i].size(), cudaMemcpyHostToDevice));
    }
    if (!h->d_ones) {
      h->n_ones = static_cast<size_t>(G) * H;
      std::vector<float> ones(h->n_ones, 1.0f);
      CUDA_TRY(cudaMalloc(&h->d_ones, sizeof(float) * h->n_ones));
      CUDA_TRY(cudaMemcpy(h->d_ones, ones.data(), sizeof(float) * h->n_ones, cudaMemcpyHostToDevice));
    }
  }
  h->packed = std::move(packed);
  h->weights_loaded = true;
  return LSPG_OK;
}

int lspr_debug_packed(lspr_handle h, int which, float* dst, int64_t* count) {
  if (!h || !count) return fail(LSPG_EINVAL, "null argument");
  if (!h->weights_loaded) return fail(LSPG_ESTATE, "weights not loaded");
  if (which < 0 || which >= static_cast<int>(h->packed.size()))
    return fail(LSPG_EINVAL, "which must be in [0, %zu) (got %d)", h->packed.size(), which);
  const std::vector<float>& v = h->packed[which];
  if (!dst) { *count = static_cast<int64_t>(v.size()); return LSPG_OK; }
  if (static_cast<size_t>(*count) != v.size()) return fail(LSPG_EINVAL, "count %lld != %zu", static_cast<long long>(*count), v.size());
  if (!v.empty()) memcpy(dst, v.data(), sizeof(float) * v.size());
  return LSPG_OK;
}

// Workspace layout (floats, every block 64-float aligned).  APC: xproj [T][3H], two layer buffers [T][H].
// MOUTH (T = n/2 LSTM steps): two MLP buffers [T][max(D, 512)], xproj [T][4*256], two LSTM buffers [T][256].
static size_t workspace_floats(const lspr_ctx* h, int n_rows, size_t off[5]) {
  size_t T, sz[5];
  int nb;
  if (h->cfg.kind == LSPR_APC) {
    T = static_cast<size_t>(n_rows);
    sz[0] = T * h->G * h->H; sz[1] = sz[2] = T * h->H; nb = 3;
  } else {
    T = static_cast<size_t>(n_rows / 2);
    const size_t w = std::max(h->cfg.input_dim, kFcW);
    sz[0] = sz[1] = T * w; sz[2] = T * h->G * h->H; sz[3] = sz[4] = T * h->H; nb = 5;
  }
  size_t total = 0;
  for (int i = 0; i < nb; ++i) { off[i] = total; total += align_floats(sz[i]); }
  return total;
}

int lspr_workspace_bytes(lspr_handle h, int n_rows, size_t* bytes) {
  if (!h || !bytes) return fail(LSPG_EINVAL, "null argument");
  if (n_rows < 0) return fail(LSPG_EINVAL, "n_rows must be >= 0 (got %d)", n_rows);
  size_t off[5];
  *bytes = sizeof(float) * workspace_floats(h, n_rows, off);
  return LSPG_OK;
}

int lspr_state_bytes(lspr_handle h, size_t* bytes) {
  if (!h || !bytes) return fail(LSPG_EINVAL, "null argument");
  *bytes = sizeof(float) * static_cast<size_t>(h->L) * 2 * h->H;      // [L][2][H]: h, then c (LSTM; unused by the GRU)
  return LSPG_OK;
}

// One span of a clip: state holds the layers' h and c, carried across calls; step0 is the global step of the span's first
// row (APC) or pair (MOUTH).  A whole clip is the span from step 0.
int lspr_forward_stream(lspr_handle h, const float* in, int n_rows, int64_t step0, float* out, float* state, void* ws,
                        size_t ws_bytes, int cluster, void* stream) {
  if (!h) return fail(LSPG_EINVAL, "null handle");
  if (!state) return fail(LSPG_EINVAL, "null state");
  const lspr_config& c = h->cfg;
  const bool apc = c.kind == LSPR_APC;
  if (n_rows < 0) return fail(LSPG_EINVAL, "n_rows must be >= 0 (got %d)", n_rows);
  if (!apc && n_rows % 2) return fail(LSPG_EINVAL, "Audio2Mouth reads APC rows in pairs: n_rows must be even (got %d)", n_rows);
  if (step0 < 0 || step0 > INT32_MAX) return fail(LSPG_EINVAL, "step0 must be in [0, 2^31) (got %lld)", static_cast<long long>(step0));
  // a MOUTH span before frame_future returns no rows, so it may pass no output buffer
  if (n_rows > 0 && (!in || (!out && (apc || step0 + n_rows / 2 > c.frame_future))))
    return fail(LSPG_EINVAL, "null buffer");
  if ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(state)) % 16)
    return fail(LSPG_EINVAL, "in, out and state must be 16-byte aligned");
  size_t off[5];
  const size_t need = sizeof(float) * workspace_floats(h, n_rows, off);
  if (ws_bytes < need) return fail(LSPG_EINVAL, "workspace of %zu bytes is smaller than the %zu needed", ws_bytes, need);
  if (need && (!ws || reinterpret_cast<uintptr_t>(ws) % 256)) return fail(LSPG_EINVAL, "workspace must be non-null and 256-byte aligned");
  int cl = cluster;
  if (apc) {
    if (cl == 0) cl = h->max_clusters16 > 0 ? 16 : 8;
    if (cl != 8 && cl != 16) return fail(LSPG_EINVAL, "APC cluster must be 0, 8 or 16 (got %d)", cluster);
  } else {
    if (cl == 0) cl = 8;
    if (cl != 8) return fail(LSPG_EINVAL, "Audio2Mouth cluster must be 0 or 8 (got %d)", cluster);
  }
  if (int rc = capi::require_device<Lspr>(h->device, "lspr_forward_stream")) return rc;
  if (!h->weights_loaded) return fail(LSPG_ESTATE, "lspr_load_weights has not been called");
  if ((cl == 16 ? h->max_clusters16 : h->max_clusters8) < 1)
    return fail(LSPG_ENODEV, "a %d-CTA cluster with %zu bytes of shared memory per CTA cannot be scheduled on device %d", cl,
                 cl == 16 ? kGru16Smem : (apc ? kGru8Smem : kLstm8Smem), h->device);
  DeviceGuard g(h->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int G = h->G, H = h->H;
  if (step0 == 0) CUDA_TRY(cudaMemsetAsync(state, 0, sizeof(float) * static_cast<size_t>(h->L) * 2 * H, st));
  if (n_rows == 0) return LSPG_OK;
  float* w = static_cast<float*>(ws);
  auto P = [&](int i) { return static_cast<const float*>(h->d_packed[i]); };
  auto layer = [&](int l, const float* x, int T, float* xproj, float* dst, const float* resid) -> int {
    gemm(x, P(4 * l), h->d_ones, P(4 * l + 1), xproj, T, G * H, h->in_w[l], 0, st);
    RecParams p{xproj, P(4 * l + 2), G == 3 ? P(4 * l + 3) : nullptr, resid, dst, state + static_cast<size_t>(l) * 2 * H, T};
    return launch_rnn(h, cl, p, st);
  };
  int r;
  if (apc) {
    const int T = n_rows;
    float* xproj = w + off[0];
    float* buf[2] = {w + off[1], w + off[2]};
    const float* x = in;
    for (int l = 0; l < h->L; ++l) {
      float* dst = l + 1 == h->L ? out : buf[l & 1];
      // models/networks.py:59-65: the layer input is added where the widths match, except after the last layer
      const float* resid = (c.residual && l + 1 < h->L && h->in_w[l] == H) ? x : nullptr;
      if ((r = layer(l, x, T, xproj, dst, resid))) return r;
      x = dst;
    }
  } else {
    // One LSTM step per pair of rows: the downsample GEMM reads `in` as [n_rows / 2, 2 D] (models/audio2feature.py:65).
    const int D = c.input_dim, ff = c.frame_future, np = n_rows / 2;
    // fc runs on the global steps >= frame_future (models/audio2feature_model.py:147 drops the first frame_future)
    const int skip = static_cast<int>(std::min<int64_t>(np, std::max<int64_t>(0, ff - step0)));
    const int n_out = np - skip;
    float *m0 = w + off[0], *m1 = w + off[1], *xproj = w + off[2], *la = w + off[3], *lb = w + off[4];
    gemm(in, P(12), P(13), P(14), m0, np, D, 2 * D, 1, st);
    gemm(m0, P(15), P(16), P(17), m1, np, D, D, 0, st);
    if ((r = layer(0, m1, np, xproj, la, nullptr))) return r;
    if ((r = layer(1, la, np, xproj, lb, nullptr))) return r;
    if ((r = layer(2, lb, np, xproj, la, nullptr))) return r;
    if (n_out > 0) {
      const float* kept = la + static_cast<size_t>(skip) * kLstmH;
      gemm(kept, P(18), P(19), P(20), m0, n_out, kFcW, kLstmH, 1, st);
      gemm(m0, P(21), P(22), P(23), m1, n_out, kFcW, kFcW, 1, st);
      gemm_nt_kernel<true><<<dim3((c.out_dim + 63) / 64, (n_out + 63) / 64), 256, 0, st>>>(m1, P(24), P(25), P(26), out,
                                                                                          n_out, c.out_dim, kFcW, 0);
    }
  }
  CUDA_TRY(cudaGetLastError());
  return LSPG_OK;
}

}  // extern "C"
