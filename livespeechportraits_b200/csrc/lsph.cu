// C-ABI implementation of the Audio2Headpose generation loop (see include/lsph.h; SURVEY.md 8f row N4).
//
// Reference: models/audio2headpose_model.py:133-187 runs, per generated frame, audio_downsample over a 255-row window,
// a 255-step WaveNet (14 gated residual blocks, dilations 1..64 twice, models/networks.py:199-227 / 303-326), copies the
// 25 GMM parameters to the host, samples on the CPU (models/losses.py:68-112) and appends the sample to the history.
//
// Here:
//   * Nothing that depends only on the audio stays in the loop: audio_downsample of every audio row (two GEMMs, eval
//     BatchNorm1d folded into the first one's epilogue) and the 2 x 14 conditioning 1x1 convolutions (one GEMM,
//     [n_audio, 512] x [512, 14*256]) are computed once per call, for every audio row it is given.
//   * The WaveNet is evaluated INCREMENTALLY over absolute time t: per frame ONE new time step, each block reading its
//     own input at t and at t - dilation from a per-layer history.  This is the same function as the reference's
//     full-window forward: the receptive field of the last window position equals the window length (255), so the
//     activations that feed it never see the window's zero padding and are identical in every window that contains
//     them.  The first rf-1 steps replay window 0 (history = pre_headpose, audio row 0 repeated) with the zero padding
//     of that window; step t = i + rf - 1 emits frame i.  tests/a2h_incremental.py is the host emulator of exactly
//     this recurrence, checked against the oracle.
//   * One persistent kernel runs all steps.  A step is a chain of 2 x 14 + 4 dependent matrix-vector products
//     (114k MACs per block): latency bound, so the work of a step is spread over a thread-block CLUSTER of 8 CTAs that
//     exchange the 128-float activation vectors through distributed shared memory (two cluster barriers per block), the
//     6.4 MB of fp32 weights stream from L2 (they do not fit in shared memory), and every stage's weight rows are
//     requested before the barrier that precedes their use.  Sample_GMM runs in the same kernel with the caller's draws.
// All arithmetic is fp32 (the reference's dtype); summation order differs from ATen's, nothing else.
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/lsph.h"
#include "capi.cuh"
#include "gemm_nt.cuh"

namespace cg = cooperative_groups;
using capi::DeviceGuard;

namespace {

struct Lsph;
constexpr auto fail = capi::fail<Lsph>;

constexpr int kR = 128;          // residual = dilation channels
constexpr int kS = 256;          // skip channels
constexpr int kMaxLayers = 16;      // layers x blocks (14 for the shipped options); bounds the per-step smem prefetch
constexpr int kMaxIn = 32;
constexpr int kMaxOut = 128;

// The hoisted audio path (audio_downsample and the conditioning projections) runs on gemm_nt_kernel (csrc/gemm_nt.cuh).

// ------------------------------------------------------------------------------------------------
// The autoregressive kernel
// ------------------------------------------------------------------------------------------------
struct LoopParams {
  const float* w_start1; const float* b_start1;      // [R][in_ch], [R]
  const float* w_start2; const float* b_start2;      // [R][R], [R]
  const float* w_fg;       // [L][2R rows: filter 0..R-1, gate R..2R-1][2R: tap 0 (x[t-d]) | tap 1 (x[t])]
  const float* w_rs;       // [L][R + S rows: residual_conv then skip_conv][R]
  const float* b_rs;       // [L][R + S]
  const float* w_end1; const float* b_end1;          // [O][S], [O]
  const float* w_end2; const float* b_end2;          // [O][O], [O]
  const float* cond;       // [n_audio][L][2R]: cond_filter/gate conv of audio rows arow0 .. + their biases + filter/gate biases
  const float* h_in;           // [in_ch]: the network input of step t0 (the last sample), or null: pre_headpose
  const float* pre_headpose;   // [in_ch]
  const float* noise;          // [n frames][ndim], row i - frame0 for frame i
  const float* uniform;        // [n frames] or null
  float* hist;                 // [L][ring][R]: input of block l at absolute time t, in slot t mod ring
  float* h_out;                // [in_ch] or null: the network input after the last step
  float* out_pred;             // [n frames][ndim]
  float* out_params;           // [n frames][O] or null
  int L, in_ch, O, ndim, ncenter, gmm;
  int n_audio, arow0, frame0, rf, ff, t0, t1, ring;
  float sigma_scale;
  int dil[kMaxLayers];
};

__device__ __forceinline__ float lrelu(float v) { return v > 0.f ? v : 0.2f * v; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float dot4(const float4& a, const float4& b) {
  return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, a.w * b.w)));
}

// CL = CTAs per cluster (1 or 8), NW = warps per CTA.  Work split of a block's two stages over the cluster:
//   stage A (filter / gate convs, 2R outputs over K = 2R): CTA c owns channels [c*R/CL, (c+1)*R/CL) of BOTH filter and gate,
//                                                        so the gated activation z of its channels is local;
//   stage B (residual conv R outputs + skip conv S outputs over K = R): CTA c owns residual channels [c*R/CL, ...) and skip
//                                                        channels [c*S/CL, ...); skip sums stay in the owner until the end.
template <int CL, int NW>
__global__ void __launch_bounds__(NW * 32, 1) headpose_loop_kernel(const LoopParams p) {
  constexpr int kRc = kR / CL;                 // residual / dilation channels per CTA
  constexpr int kSc = kS / CL;                 // skip channels per CTA
  constexpr int kOutA = 2 * kRc;               // stage-A outputs per CTA
  constexpr int kOutB = kRc + kSc;             // stage-B outputs per CTA
  constexpr int kRowsA = kOutA / NW;           // per warp
  constexpr int kRowsB = kOutB / NW;
  static_assert(kOutA % NW == 0 && kOutB % NW == 0, "outputs must divide over the warps");
  constexpr bool kPrefetch = (kRowsA * 2 + kRowsB) <= 12;   // weight rows kept in registers across a barrier

  cg::cluster_group cluster = cg::this_cluster();
  const unsigned crank = CL > 1 ? cluster.block_rank() : 0u;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  __shared__ __align__(16) float h_s[kMaxIn];          // current network input (history sample)
  __shared__ __align__(16) float s1_s[kR];             // start_conv1 output
  __shared__ __align__(16) float xbuf[2][kR];          // block input x (double buffered across blocks), full vector in every CTA
  __shared__ __align__(16) float xd_all[kMaxLayers][kR];   // delayed inputs x_l[t - d_l] of every block, fetched at step start
  __shared__ __align__(16) float cond_s[kMaxLayers][kOutA]; // this CTA's share of the step's conditioning terms
  __shared__ __align__(16) float fg_s[kOutA];          // this CTA's filter / gate pre-activations
  __shared__ __align__(16) float z_s[kR];              // gated activation, full vector in every CTA
  __shared__ __align__(16) float skip_acc[kSc];        // this CTA's skip channels, summed over the blocks of a step
  __shared__ __align__(16) float skip_full[kS];        // rank 0: LeakyReLU(skip) of all channels
  __shared__ __align__(16) float e1_s[kMaxOut];
  __shared__ __align__(16) float out_s[kMaxOut];

  if (tid < p.in_ch) h_s[tid] = p.h_in ? p.h_in[tid] : p.pre_headpose[tid];
  __syncthreads();

  float4 wa[kPrefetch ? kRowsA : 1][2];
  float4 wb[kPrefetch ? kRowsB : 1];
  float bb[kPrefetch ? kRowsB : 1];                // stage-B biases (lane 0 only)
  auto row_a = [&](int rr) {                       // global row of w_fg for this warp's rr-th stage-A output
    const int o = warp + NW * rr;                  // local output: [0, kRc) filter, [kRc, 2kRc) gate
    return (o < kRc) ? static_cast<int>(crank) * kRc + o : kR + static_cast<int>(crank) * kRc + (o - kRc);
  };
  auto row_b = [&](int rr) {
    const int o = warp + NW * rr;                  // local output: [0, kRc) residual, [kRc, kRc + kSc) skip
    return (o < kRc) ? static_cast<int>(crank) * kRc + o : kR + static_cast<int>(crank) * kSc + (o - kRc);
  };
  auto load_a = [&](int l) {
    if constexpr (kPrefetch) {
#pragma unroll
      for (int rr = 0; rr < kRowsA; ++rr) {
        const float4* q = reinterpret_cast<const float4*>(p.w_fg + (static_cast<size_t>(l) * 2 * kR + row_a(rr)) * (2 * kR));
        wa[rr][0] = __ldg(q + lane);
        wa[rr][1] = __ldg(q + 32 + lane);
      }
    }
  };
  auto load_b = [&](int l) {
    if constexpr (kPrefetch) {
#pragma unroll
      for (int rr = 0; rr < kRowsB; ++rr) {
        wb[rr] = __ldg(reinterpret_cast<const float4*>(p.w_rs + (static_cast<size_t>(l) * (kR + kS) + row_b(rr)) * kR) + lane);
        bb[rr] = __ldg(p.b_rs + l * (kR + kS) + row_b(rr));
      }
    }
  };
  load_a(0);

  int cur = 0;
  for (int t = p.t0; t < p.t1; ++t) {
    const bool emit = t >= p.rf - 1;
    int arow = t + p.ff - (p.rf - 1);                  // absolute audio row, the first rf - 1 steps replay row 0 ...
    arow = (arow < 0 ? 0 : arow) - p.arow0;            // ... relative to the first row given (the host checks coverage)
    arow = arow < 0 ? 0 : (arow > p.n_audio - 1 ? p.n_audio - 1 : arow);
    // ---- off the critical path: the delayed inputs of every block (written >= 1 step ago) and this step's conditioning terms
    for (int idx = tid; idx < p.L * kR; idx += NW * 32) {
      const int l = idx / kR, k = idx - l * kR;
      const int td = t - p.dil[l];
      xd_all[l][k] = (td >= 0) ? p.hist[(static_cast<size_t>(l) * p.ring + (td & (p.ring - 1))) * kR + k] : 0.f;  // zero padding of window 0
    }
    for (int idx = tid; idx < p.L * kOutA; idx += NW * 32) {
      const int l = idx / kOutA, o = idx - l * kOutA;
      const int row = (o < kRc) ? static_cast<int>(crank) * kRc + o : kR + static_cast<int>(crank) * kRc + (o - kRc);
      cond_s[l][o] = __ldg(p.cond + (static_cast<size_t>(arow) * p.L + l) * (2 * kR) + row);
    }
    // ---- start convs (every CTA computes the full vector; 18k MACs)
    if (tid < kR) {
      float a = p.b_start1[tid];
      const float* w = p.w_start1 + tid * p.in_ch;
      for (int k = 0; k < p.in_ch; ++k) a = fmaf(w[k], h_s[k], a);
      s1_s[tid] = lrelu(a);
    }
    if (tid < kSc) skip_acc[tid] = 0.f;
    __syncthreads();
    for (int o = warp; o < kR; o += NW) {
      const float4 w = __ldg(reinterpret_cast<const float4*>(p.w_start2 + o * kR) + lane);
      const float v = warp_sum(dot4(w, reinterpret_cast<const float4*>(s1_s)[lane]));
      if (lane == 0) xbuf[cur][o] = lrelu(v + p.b_start2[o]);
    }
    __syncthreads();

    for (int l = 0; l < p.L; ++l) {
      if (crank == 0 && tid < kR) p.hist[(static_cast<size_t>(l) * p.ring + (t & (p.ring - 1))) * kR + tid] = xbuf[cur][tid];   // X[l][t]
      load_b(l);                                     // stage-B weight rows are in flight across stage A and barrier #1
      // ---- stage A: filter / gate pre-activations of this CTA's channels
      {
        const float4 xd4 = reinterpret_cast<const float4*>(xd_all[l])[lane];
        const float4 x4 = reinterpret_cast<const float4*>(xbuf[cur])[lane];
#pragma unroll
        for (int rr = 0; rr < kRowsA; ++rr) {
          const int row = row_a(rr);
          float4 w0, w1;
          if constexpr (kPrefetch) { w0 = wa[rr][0]; w1 = wa[rr][1]; }
          else {
            const float4* q = reinterpret_cast<const float4*>(p.w_fg + (static_cast<size_t>(l) * 2 * kR + row) * (2 * kR));
            w0 = __ldg(q + lane); w1 = __ldg(q + 32 + lane);
          }
          const float v = warp_sum(dot4(w0, xd4) + dot4(w1, x4));
          if (lane == 0) fg_s[warp + NW * rr] = v + cond_s[l][warp + NW * rr];
        }
      }
      __syncthreads();
      if (tid < kRc) {
        const float f = fg_s[tid], g = fg_s[kRc + tid];
        const float z = tanhf(f) * (1.0f / (1.0f + expf(-g)));                               // networks.py:321-323
        const int ch = static_cast<int>(crank) * kRc + tid;
        if constexpr (CL > 1) {
#pragma unroll
          for (int r = 0; r < CL; ++r) cluster.map_shared_rank(z_s, r)[ch] = z;
        } else {
          z_s[ch] = z;
        }
      }
      if constexpr (CL > 1) cluster.sync(); else __syncthreads();                            // barrier #1: z complete everywhere
      load_a(l + 1 < p.L ? l + 1 : 0);               // next block's (or next step's first) stage-A rows
      // ---- stage B: residual conv (+ x) -> next block's input; skip conv -> running skip sum
      {
        const float4 z4 = reinterpret_cast<const float4*>(z_s)[lane];
#pragma unroll
        for (int rr = 0; rr < kRowsB; ++rr) {
          const int row = row_b(rr);
          const int o = warp + NW * rr;
          if (o >= kRc && !emit) continue;           // skip sums are only needed for steps that emit a frame
          float4 w;
          float bias;
          if constexpr (kPrefetch) { w = wb[rr]; bias = bb[rr]; }
          else {
            w = __ldg(reinterpret_cast<const float4*>(p.w_rs + (static_cast<size_t>(l) * (kR + kS) + row) * kR) + lane);
            bias = __ldg(p.b_rs + l * (kR + kS) + row);
          }
          float v = warp_sum(dot4(w, z4));
          if (lane == 0) {
            v += bias;
            if (o < kRc) {
              const int ch = static_cast<int>(crank) * kRc + o;
              v += xbuf[cur][ch];                                                             // networks.py:326 (+ input)
              if constexpr (CL > 1) {
#pragma unroll
                for (int r = 0; r < CL; ++r) cluster.map_shared_rank(&xbuf[cur ^ 1][0], r)[ch] = v;
              } else {
                xbuf[cur ^ 1][ch] = v;
              }
            } else {
              skip_acc[o - kRc] += v;                                                         // networks.py:216 (skip += current_skip)
            }
          }
        }
      }
      if constexpr (CL > 1) cluster.sync(); else __syncthreads();                            // barrier #2: next x complete everywhere
      cur ^= 1;
    }

    if (emit) {
      const int i = t - (p.rf - 1) - p.frame0;       // row of the frame in this launch's noise / outputs
      // ---- LeakyReLU(skip) of every CTA's channels -> rank 0
      if (tid < kSc) {
        const float v = lrelu(skip_acc[tid]);
        if constexpr (CL > 1) cluster.map_shared_rank(skip_full, 0)[static_cast<int>(crank) * kSc + tid] = v;
        else skip_full[tid] = v;
      }
      if constexpr (CL > 1) cluster.sync(); else __syncthreads();                            // barrier #3
      if (crank == 0) {
        for (int o = warp; o < p.O; o += NW) {                                               // end_conv_1: O x S
          const float4* q = reinterpret_cast<const float4*>(p.w_end1 + o * kS);
          const float v = warp_sum(dot4(__ldg(q + lane), reinterpret_cast<const float4*>(skip_full)[lane]) +
                                   dot4(__ldg(q + 32 + lane), reinterpret_cast<const float4*>(skip_full)[32 + lane]));
          if (lane == 0) e1_s[o] = lrelu(v + p.b_end1[o]);
        }
        __syncthreads();
        if (tid < p.O) {                                                                     // end_conv_2: O x O
          float a = p.b_end2[tid];
          const float* w = p.w_end2 + tid * p.O;
          for (int k = 0; k < p.O; ++k) a = fmaf(w[k], e1_s[k], a);
          out_s[tid] = a;
          if (p.out_params) p.out_params[static_cast<size_t>(i) * p.O + tid] = a;
        }
        __syncthreads();
        // ---- Sample_GMM (models/losses.py:68-112) with the caller's draws
        __shared__ int sel_s;
        if (tid == 0) {
          int sel = 0;
          if (p.gmm && p.ncenter > 1) {
            float mx = out_s[0];
            for (int k = 1; k < p.ncenter; ++k) mx = fmaxf(mx, out_s[k]);
            float tot = 0.f;
            for (int k = 0; k < p.ncenter; ++k) tot += expf(out_s[k] - mx);
            const float u = (p.uniform ? p.uniform[i] : 0.5f) * tot;
            float cum = 0.f;
            sel = p.ncenter - 1;
            for (int k = 0; k < p.ncenter; ++k) { cum += expf(out_s[k] - mx); if (u < cum) { sel = k; break; } }
          }
          sel_s = sel;
        }
        __syncthreads();
        if (tid < p.ndim) {
          float hv;
          if (p.gmm) {
            const float mu = out_s[p.ncenter + sel_s * p.ndim + tid];
            const float sigma = __fmul_rn(expf(-out_s[p.ncenter + p.ncenter * p.ndim + sel_s * p.ndim + tid]), p.sigma_scale);
            hv = __fadd_rn(__fmul_rn(p.noise[static_cast<size_t>(i) * p.ndim + tid], sigma), mu);   // losses.py:104, no FMA contraction
          } else {
            hv = out_s[tid];
          }
          p.out_pred[static_cast<size_t>(i) * p.ndim + tid] = hv;
          if constexpr (CL > 1) {
#pragma unroll
            for (int r = 0; r < CL; ++r) cluster.map_shared_rank(h_s, r)[tid] = hv;          // audio2headpose_model.py:187
          } else {
            h_s[tid] = hv;
          }
        }
      }
      if constexpr (CL > 1) cluster.sync(); else __syncthreads();                            // barrier #4: new history sample everywhere
    }
  }
  // Every CTA read h_in before its first barrier, so it may be overwritten now.
  if (p.h_out && crank == 0 && tid < p.in_ch) p.h_out[tid] = h_s[tid];
}

struct HostTensor {
  std::vector<float> v;
  bool have = false;
};

}  // namespace

struct lsph_ctx {
  lsph_config cfg{};
  int device = -1;
  int L = 0, O = 0, rf = 0;
  int ring = 0;                      // history slots per layer: the smallest power of two above the largest dilation
  std::vector<int> dil;
  bool weights_loaded = false;
  // device weights
  float *d_w_ds0 = nullptr, *d_scale0 = nullptr, *d_shift0 = nullptr;     // audio_downsample.0 + BatchNorm fold
  float *d_w_ds3 = nullptr, *d_one = nullptr, *d_b_ds3 = nullptr;         // audio_downsample.3
  float *d_w_cond = nullptr, *d_b_cond = nullptr;                         // [L*2R][C], [L*2R]
  float *d_w_start1 = nullptr, *d_b_start1 = nullptr, *d_w_start2 = nullptr, *d_b_start2 = nullptr;
  float *d_w_fg = nullptr, *d_w_rs = nullptr, *d_b_rs = nullptr;
  float *d_w_end1 = nullptr, *d_b_end1 = nullptr, *d_w_end2 = nullptr, *d_b_end2 = nullptr;
  std::vector<float*> owned;
  std::vector<float> packed[7];      // host copies of the packed arrays (lsph_debug_packed)
};

namespace {

int upload(lsph_ctx* h, float** dst, const std::vector<float>& src) {
  if (h->device < 0) return LSPG_OK;
  if (!*dst) {
    CUDA_TRY(cudaMalloc(dst, src.size() * sizeof(float)));
    h->owned.push_back(*dst);
  }
  CUDA_TRY(cudaMemcpy(*dst, src.data(), src.size() * sizeof(float), cudaMemcpyHostToDevice));
  return LSPG_OK;
}

}  // namespace

extern "C" {

const char* lsph_last_error(void) { return capi::last_error<Lsph>().c_str(); }

int lsph_create(lsph_handle* out, const lsph_config* c, int device) {
  if (!out || !c) return fail(LSPG_EINVAL, "null argument");
  *out = nullptr;
  if (c->residual_ch != kR || c->dilation_ch != kR) return fail(LSPG_EINVAL, "residual/dilation channels must be %d (got %d/%d)", kR, c->residual_ch, c->dilation_ch);
  if (c->skip_ch != kS) return fail(LSPG_EINVAL, "skip channels must be %d (got %d)", kS, c->skip_ch);
  if (c->kernel_size != 2) return fail(LSPG_EINVAL, "kernel_size must be 2 (got %d)", c->kernel_size);
  if (c->layers < 1 || c->blocks < 1 || c->layers * c->blocks > kMaxLayers || c->layers > 20) return fail(LSPG_EINVAL, "layers x blocks out of range");
  if (c->input_ch < 1 || c->input_ch > kMaxIn) return fail(LSPG_EINVAL, "input_ch out of range [1,%d]", kMaxIn);
  if (c->ndim < 1 || c->ncenter < 1) return fail(LSPG_EINVAL, "bad GMM shape");
  if (c->ndim != c->input_ch) return fail(LSPG_EINVAL, "ndim (%d) must equal input_ch (%d): the sample is fed back as the next input", c->ndim, c->input_ch);
  const int O = c->loss_gmm ? (2 * c->ndim + 1) * c->ncenter : c->ndim;
  if (O > kMaxOut) return fail(LSPG_EINVAL, "output size %d exceeds %d", O, kMaxOut);
  if (c->apc_hidden < 64 || c->apc_hidden % 64 || c->cond_ch != c->apc_hidden)
    return fail(LSPG_EINVAL, "apc_hidden must be a multiple of 64 and equal cond_ch (got %d / %d)", c->apc_hidden, c->cond_ch);
  if (c->frame_future < 0) return fail(LSPG_EINVAL, "frame_future must be >= 0");
  std::unique_ptr<lsph_ctx> h(new lsph_ctx);
  h->cfg = *c; h->device = device; h->O = O;
  h->L = c->layers * c->blocks;
  h->rf = 1;
  for (int b = 0; b < c->blocks; ++b)
    for (int i = 0; i < c->layers; ++i) { h->dil.push_back(1 << i); h->rf += (1 << i); }      // networks.py:160-176
  h->ring = 2 << (c->layers - 1);
  cudaDeviceProp prop;
  if (int rc = capi::check_device<Lsph>(device, &prop)) return rc;
  *out = h.release();
  return LSPG_OK;
}

int lsph_receptive_field(lsph_handle h, int* out) {
  if (!h || !out) return fail(LSPG_EINVAL, "null argument");
  *out = h->rf;
  return LSPG_OK;
}

int lsph_destroy(lsph_handle h) {
  if (!h) return LSPG_OK;
  if (h->device >= 0) {
    DeviceGuard g(h->device);
    for (float* p : h->owned) cudaFree(p);
  }
  delete h;
  return LSPG_OK;
}

int lsph_load_weights(lsph_handle h, const lspg_tensor* tensors, int n) {
  if (!h || (!tensors && n > 0)) return fail(LSPG_EINVAL, "null argument");
  const lsph_config& c = h->cfg;
  capi::WeightTable<Lsph> wt(tensors, n);
  if (int rc = wt.status()) return rc;
  const int H = c.apc_hidden, C = c.cond_ch, I = c.input_ch, O = h->O, L = h->L;
  // ---- audio_downsample (models/audio2headpose.py:17-22): Linear - BatchNorm1d(eval) - LeakyReLU - Linear
  const float* w0 = wt.get("audio_downsample.0.weight", static_cast<size_t>(H) * 2 * H);
  const float* b0 = wt.get("audio_downsample.0.bias", H);
  const float* bw = wt.get("audio_downsample.1.weight", H);
  const float* bb = wt.get("audio_downsample.1.bias", H);
  const float* bm = wt.get("audio_downsample.1.running_mean", H);
  const float* bv = wt.get("audio_downsample.1.running_var", H);
  const float* w3 = wt.get("audio_downsample.3.weight", static_cast<size_t>(H) * H);
  const float* b3 = wt.get("audio_downsample.3.bias", H);
  const float* ws1 = wt.get("WaveNet.start_conv1.weight", static_cast<size_t>(kR) * I);
  const float* bs1 = wt.get("WaveNet.start_conv1.bias", kR);
  const float* ws2 = wt.get("WaveNet.start_conv2.weight", static_cast<size_t>(kR) * kR);
  const float* bs2 = wt.get("WaveNet.start_conv2.bias", kR);
  const float* we1 = wt.get("WaveNet.end_conv_1.weight", static_cast<size_t>(O) * kS);
  const float* be1 = wt.get("WaveNet.end_conv_1.bias", O);
  const float* we2 = wt.get("WaveNet.end_conv_2.weight", static_cast<size_t>(O) * O);
  const float* be2 = wt.get("WaveNet.end_conv_2.bias", O);
  if (int rc = wt.status()) return rc;
  std::vector<float> scale0(H), shift0(H), one(std::max(H, L * 2 * kR), 1.0f);
  for (int j = 0; j < H; ++j) {
    const float s = bw[j] / sqrtf(bv[j] + 1e-5f);          // BatchNorm1d eval, eps = torch default
    scale0[j] = s;
    shift0[j] = (b0[j] - bm[j]) * s + bb[j];
  }
  std::vector<float> w_fg(static_cast<size_t>(L) * 2 * kR * 2 * kR), w_rs(static_cast<size_t>(L) * (kR + kS) * kR), b_rs(static_cast<size_t>(L) * (kR + kS), 0.f);
  std::vector<float> w_cond(static_cast<size_t>(L) * 2 * kR * C), b_cond(static_cast<size_t>(L) * 2 * kR, 0.f);
  for (int l = 0; l < L; ++l) {
    const std::string p = "WaveNet.residual_blocks." + std::to_string(l) + ".";
    const float* wf = wt.get(p + "filter_conv.weight", static_cast<size_t>(kR) * kR * 2);
    const float* wg = wt.get(p + "gate_conv.weight", static_cast<size_t>(kR) * kR * 2);
    const float* wr = wt.get(p + "residual_conv.weight", static_cast<size_t>(kR) * kR);
    const float* wsk = wt.get(p + "skip_conv.weight", static_cast<size_t>(kS) * kR);
    const float* wcf = wt.get(p + "cond_filter_conv.weight", static_cast<size_t>(kR) * C);
    const float* wcg = wt.get(p + "cond_gate_conv.weight", static_cast<size_t>(kR) * C);
    const float* bcf = wt.get(p + "cond_filter_conv.bias", kR);
    const float* bcg = wt.get(p + "cond_gate_conv.bias", kR);
    const float* bf = wt.get(p + "filter_conv.bias", kR, c.use_bias != 0);
    const float* bg = wt.get(p + "gate_conv.bias", kR, c.use_bias != 0);
    const float* br = wt.get(p + "residual_conv.bias", kR, c.use_bias != 0);
    const float* bsk = wt.get(p + "skip_conv.bias", kS, c.use_bias != 0);
    if (int rc = wt.status()) return rc;
    // conv1d weight [out][in][tap]; tap 0 multiplies x[t - d], tap 1 multiplies x[t] (left zero padding, networks.py:271,307)
    for (int o = 0; o < kR; ++o)
      for (int k = 0; k < kR; ++k)
        for (int tap = 0; tap < 2; ++tap) {
          w_fg[(static_cast<size_t>(l) * 2 * kR + o) * 2 * kR + tap * kR + k] = wf[(o * kR + k) * 2 + tap];
          w_fg[(static_cast<size_t>(l) * 2 * kR + kR + o) * 2 * kR + tap * kR + k] = wg[(o * kR + k) * 2 + tap];
        }
    memcpy(&w_rs[static_cast<size_t>(l) * (kR + kS) * kR], wr, sizeof(float) * kR * kR);
    memcpy(&w_rs[(static_cast<size_t>(l) * (kR + kS) + kR) * kR], wsk, sizeof(float) * kS * kR);
    memcpy(&w_cond[static_cast<size_t>(l) * 2 * kR * C], wcf, sizeof(float) * kR * C);
    memcpy(&w_cond[(static_cast<size_t>(l) * 2 * kR + kR) * C], wcg, sizeof(float) * kR * C);
    for (int o = 0; o < kR; ++o) {
      b_cond[static_cast<size_t>(l) * 2 * kR + o] = bcf[o] + (bf ? bf[o] : 0.f);
      b_cond[static_cast<size_t>(l) * 2 * kR + kR + o] = bcg[o] + (bg ? bg[o] : 0.f);
      if (br) b_rs[static_cast<size_t>(l) * (kR + kS) + o] = br[o];
    }
    if (bsk)
      for (int o = 0; o < kS; ++o) b_rs[static_cast<size_t>(l) * (kR + kS) + kR + o] = bsk[o];
  }
  DeviceGuard g(h->device);
  if (h->device >= 0) CUDA_TRY(cudaDeviceSynchronize());
  auto vec = [](const float* p, size_t n) { return std::vector<float>(p, p + n); };
  int r2;
  if ((r2 = upload(h, &h->d_w_ds0, vec(w0, static_cast<size_t>(H) * 2 * H)))) return r2;
  if ((r2 = upload(h, &h->d_scale0, scale0))) return r2;
  if ((r2 = upload(h, &h->d_shift0, shift0))) return r2;
  if ((r2 = upload(h, &h->d_w_ds3, vec(w3, static_cast<size_t>(H) * H)))) return r2;
  if ((r2 = upload(h, &h->d_one, one))) return r2;
  if ((r2 = upload(h, &h->d_b_ds3, vec(b3, H)))) return r2;
  if ((r2 = upload(h, &h->d_w_cond, w_cond))) return r2;
  if ((r2 = upload(h, &h->d_b_cond, b_cond))) return r2;
  if ((r2 = upload(h, &h->d_w_start1, vec(ws1, static_cast<size_t>(kR) * I)))) return r2;
  if ((r2 = upload(h, &h->d_b_start1, vec(bs1, kR)))) return r2;
  if ((r2 = upload(h, &h->d_w_start2, vec(ws2, static_cast<size_t>(kR) * kR)))) return r2;
  if ((r2 = upload(h, &h->d_b_start2, vec(bs2, kR)))) return r2;
  if ((r2 = upload(h, &h->d_w_fg, w_fg))) return r2;
  if ((r2 = upload(h, &h->d_w_rs, w_rs))) return r2;
  if ((r2 = upload(h, &h->d_b_rs, b_rs))) return r2;
  if ((r2 = upload(h, &h->d_w_end1, vec(we1, static_cast<size_t>(O) * kS)))) return r2;
  if ((r2 = upload(h, &h->d_b_end1, vec(be1, O)))) return r2;
  if ((r2 = upload(h, &h->d_w_end2, vec(we2, static_cast<size_t>(O) * O)))) return r2;
  if ((r2 = upload(h, &h->d_b_end2, vec(be2, O)))) return r2;
  h->packed[0] = w_fg; h->packed[1] = w_rs; h->packed[2] = b_rs; h->packed[3] = w_cond; h->packed[4] = b_cond;
  h->packed[5] = scale0; h->packed[6] = shift0;
  h->weights_loaded = true;
  return LSPG_OK;
}

int lsph_debug_packed(lsph_handle h, int which, float* dst, int64_t count) {
  if (!h || !dst) return fail(LSPG_EINVAL, "null argument");
  if (which < 0 || which > 6) return fail(LSPG_EINVAL, "which must be 0..6");
  if (!h->weights_loaded) return fail(LSPG_ESTATE, "weights not loaded");
  if (static_cast<size_t>(count) != h->packed[which].size())
    return fail(LSPG_EINVAL, "count %lld != %zu", static_cast<long long>(count), h->packed[which].size());
  memcpy(dst, h->packed[which].data(), sizeof(float) * h->packed[which].size());
  return LSPG_OK;
}

// Workspace of the hoisted audio path for n_audio rows (floats, every block 64-float aligned): ds1, ds2 [n][H], cond [n][L][2R].
static size_t hoisted_floats(const lsph_ctx* h, int n_audio, size_t off[3]) {
  const size_t n = static_cast<size_t>(n_audio), sz[3] = {n * h->cfg.apc_hidden, n * h->cfg.apc_hidden, n * h->L * 2 * kR};
  size_t total = 0;
  for (int i = 0; i < 3; ++i) { off[i] = total; total += (sz[i] + 63) / 64 * 64; }
  return total;
}

static size_t state_floats(const lsph_ctx* h) { return static_cast<size_t>(h->L) * h->ring * kR + kMaxIn; }

int lsph_state_bytes(lsph_handle h, size_t* bytes) {
  if (!h || !bytes) return fail(LSPG_EINVAL, "null argument");
  *bytes = sizeof(float) * state_floats(h);
  return LSPG_OK;
}

int lsph_stream_workspace_bytes(lsph_handle h, int n_audio, size_t* bytes) {
  if (!h || !bytes) return fail(LSPG_EINVAL, "null argument");
  if (n_audio < 0) return fail(LSPG_EINVAL, "n_audio must be >= 0 (got %d)", n_audio);
  size_t off[3];
  *bytes = sizeof(float) * hoisted_floats(h, n_audio, off);
  return LSPG_OK;
}

int lsph_generate_stream(lsph_handle h, const float* audio_feats, int audio_row0, int n_audio, int frame0, int n_frames,
                         const float* pre_headpose, const float* noise, const float* uniform, float sigma_scale,
                         float* out_pred, float* out_params, float* state, void* ws, size_t ws_bytes, int cluster,
                         void* stream) {
  if (!h) return fail(LSPG_EINVAL, "null handle");
  const lsph_config& c = h->cfg;
  if (!state) return fail(LSPG_EINVAL, "null state");
  if (frame0 < 0 || n_frames < 0 || audio_row0 < 0 || n_audio < 0)
    return fail(LSPG_EINVAL, "frame0, n_frames, audio_row0 and n_audio must be >= 0 (got %d, %d, %d, %d)", frame0, n_frames,
                audio_row0, n_audio);
  const int64_t lo = frame0 == 0 ? 0 : static_cast<int64_t>(frame0) + c.frame_future;   // frame 0 also replays rows 0 ..
  const int64_t hi = static_cast<int64_t>(frame0) + n_frames + c.frame_future;           // exclusive
  if (hi + h->rf > INT32_MAX) return fail(LSPG_EINVAL, "frame0 + n_frames is too large");
  if (n_frames > 0 && (audio_row0 > lo || static_cast<int64_t>(audio_row0) + n_audio < hi))
    return fail(LSPG_EINVAL, "frames %d .. %d need audio rows %lld .. %lld, the rows given are %d .. %lld", frame0,
                frame0 + n_frames - 1, static_cast<long long>(lo), static_cast<long long>(hi - 1), audio_row0,
                static_cast<long long>(audio_row0) + n_audio - 1);
  if (n_frames > 0 && (!audio_feats || !pre_headpose || !out_pred)) return fail(LSPG_EINVAL, "null buffer");
  if (n_frames > 0 && c.loss_gmm && !noise) return fail(LSPG_EINVAL, "noise is required for the GMM loss (pass zeros for sigma_scale 0)");
  if (reinterpret_cast<uintptr_t>(state) % 16) return fail(LSPG_EINVAL, "state must be 16-byte aligned");
  size_t off[3];
  const size_t need = n_frames > 0 ? sizeof(float) * hoisted_floats(h, n_audio, off) : 0;
  if (ws_bytes < need) return fail(LSPG_EINVAL, "workspace of %zu bytes is smaller than the %zu needed", ws_bytes, need);
  if (need && (!ws || reinterpret_cast<uintptr_t>(ws) % 256)) return fail(LSPG_EINVAL, "workspace must be non-null and 256-byte aligned");
  if (cluster == 0) cluster = 8;
  if (cluster != 1 && cluster != 8) return fail(LSPG_EINVAL, "cluster must be 1 or 8 (got %d)", cluster);
  if (int rc = capi::require_device<Lsph>(h->device, "lsph_generate_stream")) return rc;
  if (!h->weights_loaded) return fail(LSPG_ESTATE, "lsph_load_weights has not been called");
  if (n_frames == 0) return LSPG_OK;
  DeviceGuard g(h->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int H = c.apc_hidden, L = h->L;
  float* w = static_cast<float*>(ws);
  float *ds1 = w + off[0], *ds2 = w + off[1], *cond = w + off[2];
  float* h_state = state + static_cast<size_t>(L) * h->ring * kR;     // after the history ring
  // ---- hoisted audio path: downsample every row given, project it for every block
  const dim3 blk(256);
  const int mt = (n_audio + 63) / 64;
  gemm_nt_kernel<><<<dim3(H / 64, mt), blk, 0, st>>>(audio_feats, h->d_w_ds0, h->d_scale0, h->d_shift0, ds1, n_audio, H, 2 * H, 1);
  gemm_nt_kernel<><<<dim3(H / 64, mt), blk, 0, st>>>(ds1, h->d_w_ds3, h->d_one, h->d_b_ds3, ds2, n_audio, H, H, 0);
  gemm_nt_kernel<><<<dim3(L * 2 * kR / 64, mt), blk, 0, st>>>(ds2, h->d_w_cond, h->d_one, h->d_b_cond, cond, n_audio, L * 2 * kR, H, 0);
  CUDA_TRY(cudaGetLastError());
  // ---- the loop over frames frame0 .. frame0 + n_frames - 1: absolute steps from t0 = frame0 + rf - 1, or from 0 with
  // the warm-up when frame0 == 0
  LoopParams p;
  memset(&p, 0, sizeof(p));
  p.w_start1 = h->d_w_start1; p.b_start1 = h->d_b_start1; p.w_start2 = h->d_w_start2; p.b_start2 = h->d_b_start2;
  p.w_fg = h->d_w_fg; p.w_rs = h->d_w_rs; p.b_rs = h->d_b_rs;
  p.w_end1 = h->d_w_end1; p.b_end1 = h->d_b_end1; p.w_end2 = h->d_w_end2; p.b_end2 = h->d_b_end2;
  p.cond = cond; p.h_in = frame0 > 0 ? h_state : nullptr; p.pre_headpose = pre_headpose;
  p.noise = noise; p.uniform = uniform;
  p.hist = state; p.h_out = h_state; p.out_pred = out_pred; p.out_params = out_params;
  p.L = L; p.in_ch = c.input_ch; p.O = h->O; p.ndim = c.ndim; p.ncenter = c.ncenter; p.gmm = c.loss_gmm;
  p.n_audio = n_audio; p.arow0 = audio_row0; p.frame0 = frame0; p.rf = h->rf; p.ff = c.frame_future;
  p.t0 = frame0 == 0 ? 0 : frame0 + h->rf - 1; p.t1 = frame0 + n_frames + h->rf - 1; p.ring = h->ring;
  p.sigma_scale = sigma_scale;
  for (int l = 0; l < L; ++l) p.dil[l] = h->dil[l];
  if (cluster == 8) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(8); cfg.blockDim = dim3(16 * 32); cfg.dynamicSmemBytes = 0; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 8; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    CUDA_TRY(cudaLaunchKernelEx(&cfg, headpose_loop_kernel<8, 16>, p));
  } else {
    headpose_loop_kernel<1, 32><<<1, 32 * 32, 0, st>>>(p);
    CUDA_TRY(cudaGetLastError());
  }
  return LSPG_OK;
}

}  // extern "C"
