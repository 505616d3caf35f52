// Fused 3x3 convolution as an implicit GEMM on Hopper tensor cores (wgmma, sm_90a).
//
// One kernel family serves every conv of the Res-UNet generator
// (reference: models/networks.py:585-675; SURVEY.md section 2a K1..K5):
//
//   D[128 pixels x BN channels] (+)= A[128 pixels x 64 ch] * B[BN x 64 ch]^T      per K block
//
//   * A K block = (tap, concat source, 64-channel chunk).  The A tile of a tap is the output tile's pixel
//     patch shifted by (dx, dy): ONE 5-D TMA box {64 ch, TW, TH, NB, 1 limb} out of the NHWC activation
//     tensor; out-of-range coordinates are zero-filled by TMA, which is the conv's zero padding.
//   * stride-2 convs read through four parity views of the input (base offset + doubled strides), the
//     nearest-x2 upsample is folded into four output phases with 2x2 pre-summed taps whose results are
//     stored with stride 2 in x and y, and torch.cat([skip, deeper]) is two K ranges fed from two tensor maps -
//     so upsample, concat, padding and stride never touch HBM as separate passes.
//   * B tiles come from a packed weight tensor [phase*limb][Cout][K] (K-major), same 128B-swizzled layout.
//   * Warp specialisation: warpgroup 0 = TMA producer (one warp), warpgroups 1 and 2 = consumers issuing
//     wgmma.m64nBNk16 with fp32 accumulators in registers, then running the epilogue from those registers: folded
//     eval-BatchNorm scale/shift in fp32, residual, ReLU, 16-bit (hi, lo) NHWC stores.  The tail variant (patch kernel
//     only) applies tanh and scatters fp32 NCHW or uint8 HWC directly.
//     conv_umma_kernel: consumer w owns rows [64w, 64w+64) of every tile.  conv_patch_kernel: ping-pong, consumer w
//     owns every other tile (all 128 rows, two accumulators), so its epilogue runs under the other one's MMAs.
//   * NL = 2 ("parity" precision): activations and weights are split into fp16 hi + lo limbs; each K step issues
//     hi*hi + hi*lo + lo*hi into one accumulator (22 mantissa bits per operand, fp32 accumulate) and the epilogue writes
//     both limbs.  NL = 1 ("fast"): one bf16 limb, one MMA per K step.
//
// Two conv kernels: conv_umma_kernel (one TMA box per tap; stride-2 convs and grids narrower than 8 or shorter than 16)
// and conv_patch_kernel (one halo patch per chunk; every other layer including the tail, optionally as a 2-CTA cluster
// that multicasts the weight tiles).  Both are persistent: each CTA walks tiles blockIdx.x, +gridDim.x, ...  Both, and the
// split-K finisher splitk_reduce_kernel, apply the regular epilogue through one helper, epilogue_pair.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include "ptx.cuh"

namespace lspg {

constexpr int kTileM = 128;                 // output pixels per tile (two wgmma M=64 halves)
constexpr int kChunk = 64;                  // channels per K block = 128 bytes of 16-bit values = one swizzle row
constexpr int kATile = kTileM * 128;        // bytes of one A tile
constexpr int kMaxTaps = 9;
constexpr int kThreads = 384;               // producer warpgroup + 2 consumer warpgroups
constexpr int kSmemBudget = 227 * 1024;

// Division by a launch-time constant as multiply-high + shift (dividend < 2^31): decode_tile runs between two tiles of
// the persistent loops, where ~9 hardware integer divisions cost more than a thousand cycles.
struct FastDiv {
  uint32_t mul, shr, d;
};
inline FastDiv make_fast_div(uint32_t d) {
  FastDiv f;
  f.d = d; f.mul = 0; f.shr = 0;
  if (d > 1) {
    uint32_t l = 0;
    while ((1u << l) < d) ++l;
    const uint64_t pw = 31 + l;
    f.mul = static_cast<uint32_t>(((1ull << pw) + d - 1) / d);
    f.shr = static_cast<uint32_t>(pw - 32);
  }
  return f;
}
__device__ __forceinline__ int fast_div(int n, const FastDiv& f) {
  return f.d == 1 ? n : static_cast<int>(__umulhi(static_cast<uint32_t>(n), f.mul) >> f.shr);
}

struct alignas(64) ConvParams {
  // Everything the epilogue and the tile decode read every tile comes first (kernel parameters are read through the
  // per-SM constant cache), the producer scalars and tap tables follow, the tensor maps (read by the TMA unit) come last.
  // ---- epilogue + tile decode (hot)
  const float* scale;        // folded BatchNorm (or 1/0), [Cout_pad]
  const float* shift;
  __nv_bfloat16* out_ptr;         // output tensor (NHWC), limb 0; written directly by the epilogue
  const __nv_bfloat16* res_ptr;   // residual tensor (NHWC, same grid as the output), limb 0; read directly by the epilogue
  long long out_limb_stride;      // elements between limbs
  long long res_limb_stride;      // elements between limbs
  float* out_f32;            // tail only: fp32 NCHW [B, 3, 2*hs, 2*ws]
  uint8_t* out_u8;           // tail only, optional: uint8 HWC image [B, 2*hs, 2*ws, 3] = util.tensor2im fused (then out_f32 is unused)
  float* partial;            // split-K partial tiles (see n_split)
  unsigned long long* trace; // debug: per-CTA clock64 stamps (null in production), see kTraceSlots
  int32_t out_channels, res_channels;
  int32_t out_up;            // the sampling grid is the source of a folded x2 upsample (phase tc.z -> (2y+py, 2x+px))
  int32_t relu, has_res;
  int32_t batch, hs, ws;     // sampling-grid extent (tail epilogue addressing)
  int32_t tw_log2, th_log2;  // tile = TW x TH pixels x NB images, TW*TH*NB = 128
  int32_t total_tiles;       // tiles_x*tiles_y*tiles_n * n_tiles * n_phases * n_split
  // split-K: the K loop (per-tap kernel: K blocks; patch kernel: (source, chunk) items) is cut into n_split ranges of
  // split_len; tile index = split * tiles_per_split + tile.  Each CTA writes its raw fp32 accumulator tile to
  // partial[tile_index][128][BN]; splitk_reduce_kernel sums the splits and applies the epilogue.
  int32_t n_split, tiles_per_split;
  int32_t n_tiles;           // Cout_pad / BN
  int32_t tiles_x, tiles_y, tiles_n;
  int32_t n_phases;
  int32_t trace_skip;        // debug: the trace records local tiles [trace_skip, trace_skip + kTraceTiles)
  FastDiv fd_tps, fd_m_tiles, fd_n_tiles, fd_tiles_x, fd_tiles_y;   // divisions of decode_tile (tiles_per_split, ...)
  // ---- MMA issue + TMA producer
  int32_t n_taps, n_src;
  int32_t chunks[2];         // 64-channel chunks per concat source
  int32_t split_len;
  // patch mode: one halo patch {64 ch, patch_w, patch_h} per (tile, source, chunk) whose origin is the tile origin +
  // (patch_dx0, patch_dy0)[phase]; every tap is a row offset inside the patch.
  int32_t patch_w, patch_h;
  int8_t patch_dx0[4], patch_dy0[4];
  int16_t tap_row[4][kMaxTaps];  // [phase][tap] -> first patch row of the tap's shifted A tile
  int8_t tap_map[4][kMaxTaps];   // [phase][tap] -> index into a[] (added to the concat source index)
  int8_t tap_dx[4][kMaxTaps];
  int8_t tap_dy[4][kMaxTaps];
  // ---- tensor maps
  CUtensorMap a[4];          // activation views: [parity or concat source], dims {C, X, Y, N, limb}
  CUtensorMap w;             // packed weights, dims {K, Cout_pad, limb*n_phases + phase} (patch kernel: {kc, Cout, tap, limb*phase})
};

// Shared-memory regions after the operand rings: barriers, then (patch kernel, tail) the accumulator staging of the tail
// epilogue, one tile per consumer warpgroup (its consumers own whole tiles).
constexpr int kBarBytes = 1024;
constexpr int kTailStride = 17;                                      // floats per staged tail row (16 + 1: no bank conflicts)
template <bool TAIL>
struct AuxCfg {
  static constexpr int kTailBytes = TAIL ? 2 * kTileM * kTailStride * 4 : 0;
  static constexpr int kBytes = kBarBytes + kTailBytes;
};

template <int BN, int NL>
struct ConvCfg {
  static constexpr int kBTile = BN * 128;
  static constexpr int kStage = NL * (kATile + kBTile);
  static constexpr int kAvail = kSmemBudget - 1024 /*alignment slack*/ - kBarBytes;
  static constexpr int kStagesRaw = kAvail / kStage;
  static constexpr int kStages = kStagesRaw > 8 ? 8 : kStagesRaw;
  static constexpr int kSmemBytes = 1024 + kStages * kStage + kBarBytes;
  static_assert(kStages >= 2, "pipeline needs at least two stages");
  static_assert(BN == 64 || BN == 128, "instantiated N tiles");
};

// Debug trace layout per CTA: [0] kernel entry, [1] prologue done, [2]/[3] globaltimer (ns) at entry/exit, then per
// local tile i (up to kTraceTiles): base = 4 + 8*i: +0 consumers start the tile, +1 first stage landed, +2 last MMA
// retired, +3 epilogue done, +6 PROD first load of the tile issued, +7 PROD last load issued.  +0..+3 are written by
// the leader thread of the warpgroup that runs the tile's MMAs (the patch kernel: the tile's owner, +0 once the
// other warpgroup has issued the previous tile; the per-tap kernel: warpgroup 1).
constexpr int kTraceTiles = 12;
constexpr int kTraceSlots = 4 + 8 * kTraceTiles + 4;   // tail: [+0] clock64 at kernel exit

struct TileCoord {
  int z, nt, x0, y0, n0, split;
};

__device__ __forceinline__ void trace_stamp(const ConvParams& p, int slot) {
  if (p.trace != nullptr && slot < kTraceSlots) p.trace[static_cast<size_t>(blockIdx.x) * kTraceSlots + slot] = clock64();
}
__device__ __forceinline__ void trace_time(const ConvParams& p, bool at_exit) {
  if (p.trace != nullptr) {
    unsigned long long ns;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(ns));
    unsigned long long* t = p.trace + static_cast<size_t>(blockIdx.x) * kTraceSlots;
    t[at_exit ? 3 : 2] = ns;
    if (at_exit) t[4 + 8 * kTraceTiles] = clock64();
  }
}
__device__ __forceinline__ void trace_tile(const ConvParams& p, int lt, int k) {
  if (p.trace != nullptr) {
    const int i = lt - p.trace_skip;
    if (i >= 0 && i < kTraceTiles) p.trace[static_cast<size_t>(blockIdx.x) * kTraceSlots + 4 + 8 * i + k] = clock64();
  }
}

__device__ __forceinline__ TileCoord decode_tile(const ConvParams& p, int t) {
  TileCoord c;
  c.split = fast_div(t, p.fd_tps);
  t -= c.split * p.tiles_per_split;
  const int r = fast_div(t, p.fd_m_tiles);
  const int mt = t - r * static_cast<int>(p.fd_m_tiles.d);
  c.z = fast_div(r, p.fd_n_tiles);
  c.nt = r - c.z * p.n_tiles;
  const int r2 = fast_div(mt, p.fd_tiles_x);
  const int tx = mt - r2 * p.tiles_x;
  const int tn = fast_div(r2, p.fd_tiles_y);
  const int ty = r2 - tn * p.tiles_y;
  c.x0 = tx << p.tw_log2;
  c.y0 = ty << p.th_log2;
  c.n0 = tn << (7 - p.tw_log2 - p.th_log2);
  return c;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);   // .x = lo (low 16 bits), .y = hi
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t u) { return __uint_as_float(u & 0xFFFF0000u); }

// 16-bit operand formats.  FAST (one limb) keeps bf16 (north_star's "bf16 in / fp32 accum").  PARITY (two limbs) uses fp16:
// hi = fp16(v), lo = fp16(v - hi) carry 22 mantissa bits where two bf16 limbs carry 16, at the same tensor cost
// (wgmma takes either format) - oracle/precision_study.py: 4.3e-5 instead of 2.2e-4 on the hard case.  The range is
// fp16's: conversions saturate at +-65504 instead of producing infinities (activations of this network are O(1..100)).
// F16 = (NL == 2) everywhere.
template <bool F16>
__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
  if constexpr (F16) {
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));     // upper half <- first source
    return r;
  } else {
    return pack_bf16x2(lo, hi);
  }
}
template <bool F16>
__device__ __forceinline__ float unpack_lo(uint32_t u) {
  if constexpr (F16) return __half2float(__ushort_as_half(static_cast<unsigned short>(u & 0xFFFFu)));
  else return bf16_lo(u);
}
template <bool F16>
__device__ __forceinline__ float unpack_hi(uint32_t u) {
  if constexpr (F16) return __half2float(__ushort_as_half(static_cast<unsigned short>(u >> 16)));
  else return bf16_hi(u);
}

// Pixel of tile row `row` (rows are x-fastest, then y, then image).
__device__ __forceinline__ void row_pixel(const ConvParams& p, const TileCoord& tc, int row, int& n, int& y, int& x) {
  x = tc.x0 + (row & ((1 << p.tw_log2) - 1));
  y = tc.y0 + ((row >> p.tw_log2) & ((1 << p.th_log2) - 1));
  n = tc.n0 + (row >> (p.tw_log2 + p.th_log2));
}

// Channel 0 of sampling-grid pixel (n, y, x) in the NHWC output (limb 0): with a folded x2 upsample, phase tc.z of it.
__device__ __forceinline__ __nv_bfloat16* out_pixel(const ConvParams& p, const TileCoord& tc, int n, int y, int x) {
  const int oh = p.out_up ? 2 * p.hs : p.hs, ow = p.out_up ? 2 * p.ws : p.ws;
  const int oy = p.out_up ? 2 * y + (tc.z >> 1) : y, ox = p.out_up ? 2 * x + (tc.z & 1) : x;
  return p.out_ptr + ((static_cast<size_t>(n) * oh + oy) * ow + ox) * p.out_channels;
}

// Regular epilogue of channel pair j of a pixel, whose channels start at out[kStride * j] (limb 0) and, in PARITY, at
// out[out_limb_stride + kStride * j]: folded BatchNorm fma, the residual's limbs in limb order (rw[l][j] = the pair's
// word of limb l, read only if p.has_res), ReLU, then the 16-bit hi word and the lo word of the remainder y - hi.
template <int kStride, int NL, int M>
__device__ __forceinline__ void epilogue_pair(const ConvParams& p, float a0, float a1, float2 s2, float2 f2,
                                              const uint32_t (&rw)[NL][M], int j, __nv_bfloat16* out) {
  float y0 = fmaf(a0, s2.x, f2.x);
  float y1 = fmaf(a1, s2.y, f2.y);
  if (p.has_res) {
#pragma unroll
    for (int l = 0; l < NL; ++l) {
      y0 += unpack_lo<NL == 2>(rw[l][j]);
      y1 += unpack_hi<NL == 2>(rw[l][j]);
    }
  }
  if (p.relu) { y0 = fmaxf(y0, 0.0f); y1 = fmaxf(y1, 0.0f); }
  const uint32_t o = pack2<NL == 2>(y0, y1);
  *reinterpret_cast<uint32_t*>(out + kStride * j) = o;
  if (NL == 2)
    *reinterpret_cast<uint32_t*>(out + p.out_limb_stride + kStride * j) = pack2<true>(y0 - unpack_lo<true>(o), y1 - unpack_hi<true>(o));
}

// Consumer epilogue of the 64 tile rows [rb, rb+64) held by one m64nBN accumulator of the calling warpgroup.
// Thread layout of the m64nBN accumulator: rows r0 = 16*warp + lane/4 and r0 + 8, columns 8j + 2*(lane%4) and +1
// (d[4j], d[4j+1] for r0; d[4j+2], d[4j+3] for r0 + 8).
// Modes: split-K partial (fp32 rows to the global scratch), tail (via shared memory: tanh and
// the NCHW / uint8 scatter want all 12 columns of a pixel in one thread), and the regular epilogue.
// Tail only: `tail_stg` is this call's 64-row staging region, `tail_bar` the calling warpgroup's named barrier.
template <int BN, int NL, bool TAIL>
__device__ __forceinline__ void epilogue_regs(const ConvParams& p, const float (&acc)[BN / 2], const TileCoord& tc, int t, int rb,
                                              float* tail_stg, int tail_bar) {
  const int wtid = threadIdx.x & 127;
  const int warp = wtid >> 5, lane = wtid & 31;
  const int r0 = rb + warp * 16 + (lane >> 2);
  const int c0 = 2 * (lane & 3);
  if constexpr (TAIL) {
    // ---- tail: 16 columns = 4 phases x 3 channels (+4 pad); tanh; fp32 NCHW scatter or fused tensor2im
    float* stg = tail_stg;
    ptx::named_bar_sync(tail_bar, 128);                   // the previous tile's rows have been read
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float* s = stg + (r0 - rb + 8 * h) * kTailStride + 8 * j + c0;
        s[0] = acc[4 * j + 2 * h];
        s[1] = acc[4 * j + 2 * h + 1];
      }
    ptx::named_bar_sync(tail_bar, 128);
    if (wtid >= 64) return;
    const int row = rb + wtid;
    const float* v = stg + wtid * kTailStride;
    int pn, py_, px_;
    row_pixel(p, tc, row, pn, py_, px_);
    if (pn >= p.batch || py_ >= p.hs || px_ >= p.ws) return;
    const int oh = 2 * p.hs, ow = 2 * p.ws;
    if (p.out_u8 != nullptr) {
      // fused util/util.py:tensor2im (reference lines 33-42): (x + 1) / 2 * 255 in fp32, clip to [0,255], truncate to
      // uint8, CHW -> HWC.  This thread owns output pixels (2y+py, 2x+px): per py, 2 pixels x 3 channels = 6 bytes.
#pragma unroll
      for (int py = 0; py < 2; ++py) {
        uint8_t b[6];
#pragma unroll
        for (int px = 0; px < 2; ++px)
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            const int col = (py * 2 + px) * 3 + c;
            const float vf = tanhf(v[col] * __ldg(p.scale + col) + __ldg(p.shift + col));
            float u = __fmul_rn(__fmul_rn(__fadd_rn(vf, 1.0f), 0.5f), 255.0f);
            u = fminf(fmaxf(u, 0.0f), 255.0f);
            b[px * 3 + c] = static_cast<uint8_t>(static_cast<int>(u));
          }
        uint8_t* dst = p.out_u8 + ((static_cast<size_t>(pn) * oh + (2 * py_ + py)) * ow + 2 * px_) * 3;
        uint16_t* d16 = reinterpret_cast<uint16_t*>(dst);          // 6-byte aligned: 2x * 3 is even
        d16[0] = static_cast<uint16_t>(b[0] | (b[1] << 8));
        d16[1] = static_cast<uint16_t>(b[2] | (b[3] << 8));
        d16[2] = static_cast<uint16_t>(b[4] | (b[5] << 8));
      }
    } else {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
#pragma unroll
        for (int py = 0; py < 2; ++py) {
          const int c0_ = (py * 2 + 0) * 3 + c, c1_ = (py * 2 + 1) * 3 + c;
          float2 o;
          o.x = tanhf(v[c0_] * __ldg(p.scale + c0_) + __ldg(p.shift + c0_));
          o.y = tanhf(v[c1_] * __ldg(p.scale + c1_) + __ldg(p.shift + c1_));
          float* dst = p.out_f32 + ((static_cast<size_t>(pn) * 3 + c) * oh + (2 * py_ + py)) * ow + 2 * px_;
          *reinterpret_cast<float2*>(dst) = o;
        }
      }
    }
  } else {
    if (p.n_split > 1) {
      // ---- split-K partial: raw fp32 accumulator rows -> partial[t][row][BN]
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float* dst = p.partial + (static_cast<size_t>(t) * kTileM + r0 + 8 * h) * BN + c0;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
          *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      }
      return;
    }
    // ---- regular: scale/shift (+ residual) + ReLU, 16-bit (hi, lo), written straight to the NHWC output
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      int pn, py_, px_;
      row_pixel(p, tc, r0 + 8 * h, pn, py_, px_);
      if (pn >= p.batch || py_ >= p.hs || px_ >= p.ws) continue;
      __nv_bfloat16* out_row = out_pixel(p, tc, pn, py_, px_) + tc.nt * BN + c0;
      const __nv_bfloat16* res_row =
          p.has_res ? p.res_ptr + ((static_cast<size_t>(pn) * p.hs + py_) * p.ws + px_) * p.res_channels + tc.nt * BN + c0 : nullptr;
      const float* sc = p.scale + tc.nt * BN + c0;
      const float* sf = p.shift + tc.nt * BN + c0;
      // residual words of the whole row first (independent loads in flight), then the math
      uint32_t rw[NL][BN / 8];
      if (p.has_res) {
#pragma unroll
        for (int l = 0; l < NL; ++l)
#pragma unroll
          for (int j = 0; j < BN / 8; ++j)
            rw[l][j] = __ldg(reinterpret_cast<const unsigned int*>(res_row + l * p.res_limb_stride + 8 * j));
      }
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const float2 s2 = __ldg(reinterpret_cast<const float2*>(sc + 8 * j));
        const float2 f2 = __ldg(reinterpret_cast<const float2*>(sf + 8 * j));
        epilogue_pair<8>(p, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], s2, f2, rw, j, out_row);
      }
    }
  }
}

// Release of a consumed ring stage: one arrive per consuming warpgroup on the stage's empty barrier in every CTA of `CL`
// (a stage filled by multicast is refilled only after every CTA that received it is done with it).
template <int CL>
__device__ __forceinline__ void release_stage(uint64_t* bar) {
  if constexpr (CL == 1) ptx::mbar_arrive(bar);
  else {
#pragma unroll
    for (int c = 0; c < CL; ++c) ptx::mbar_arrive_cluster(bar, static_cast<uint32_t>(c));
  }
}

template <int BN, int NL>
__global__ void __launch_bounds__(kThreads, 1) conv_umma_kernel(const __grid_constant__ ConvParams p) {
  using Cfg = ConvCfg<BN, NL>;
  const int t0 = static_cast<int>(blockIdx.x), tstep = static_cast<int>(gridDim.x);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* aux = smem + Cfg::kStages * Cfg::kStage;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(aux);   // [kStages]
  uint64_t* empty_bar = full_bar + Cfg::kStages;           // [kStages]

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);   // provably warp-uniform
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) { trace_stamp(p, 0); trace_time(p, false); }

  if (warp == 0 && lane == 0) {
    for (int i = 0; i < 4; ++i) ptx::prefetch_tmap(&p.a[i]);
    ptx::prefetch_tmap(&p.w);
    for (int i = 0; i < Cfg::kStages; ++i) {
      ptx::mbar_init(&full_bar[i], 1);
      ptx::mbar_init(&empty_bar[i], 2);    // one arrive per consumer warpgroup
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  ptx::pdl_launch_dependents();   // the next kernel may start its prologue; it waits (pdl_wait) before touching our output
  if (threadIdx.x == 0) trace_stamp(p, 1);

  int kb_per_tap = 0;
  for (int s = 0; s < p.n_src; ++s) kb_per_tap += p.chunks[s];
  const int num_kb = p.n_taps * kb_per_tap;

  if (warp == 0) {
    // ===================================================================== TMA producer
    // Weights are never written by a kernel, so the weight tiles of this CTA's first K blocks (a whole ring of them) are
    // requested BEFORE the programmatic-dependency wait: they stream from HBM/L2 while the previous layer is still
    // finishing.  At batch 1 the layers below 16x16 are one tile of 4-9 K blocks per CTA - their whole weight share.
    int pre = 0;
    if (t0 < p.total_tiles) {
      const TileCoord tc = decode_tile(p, t0);
      const int kb0 = tc.split * p.split_len;
      const int kb1 = (kb0 + p.split_len < num_kb) ? kb0 + p.split_len : num_kb;
      pre = (kb1 - kb0 < Cfg::kStages) ? kb1 - kb0 : Cfg::kStages;
      if (ptx::elect_one()) {
        for (int i = 0; i < pre; ++i) {          // first use of stages 0..pre-1: no empty-barrier wait needed
          uint8_t* st = smem + i * Cfg::kStage;
          ptx::mbar_expect_tx(&full_bar[i], Cfg::kStage);
#pragma unroll
          for (int l = 0; l < NL; ++l)
            ptx::tma_load_3d(&p.w, &full_bar[i], st + NL * kATile + l * Cfg::kBTile, (kb0 + i) * kChunk, tc.nt * BN,
                             l * p.n_phases + tc.z);
        }
      }
      __syncwarp();
    }
    ptx::pdl_wait();                // activations are written by the previous kernel
    int stage = 0;
    uint32_t phase = 0;
    int issued = 0;                 // K blocks issued so far by this CTA (the first `pre` already have their weight tiles)
    int lt = 0;
    for (int t = t0; t < p.total_tiles; t += tstep, ++lt) {
      const TileCoord tc = decode_tile(p, t);
      const int kb0 = tc.split * p.split_len;
      const int kb1 = (kb0 + p.split_len < num_kb) ? kb0 + p.split_len : num_kb;
      if (lane == 0) trace_tile(p, lt, 6);
      for (int kb = kb0; kb < kb1; ++kb, ++issued) {
        const int tap = kb / kb_per_tap;
        const int rem = kb - tap * kb_per_tap;
        const int s = (rem < p.chunks[0]) ? 0 : 1;
        const int c = s ? rem - p.chunks[0] : rem;
        const int amap = p.tap_map[tc.z][tap];
        const int xx = tc.x0 + p.tap_dx[tc.z][tap];
        const int yy = tc.y0 + p.tap_dy[tc.z][tap];
        const bool early = issued < pre;
        if (!early) ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
        if (ptx::elect_one()) {
          uint8_t* st = smem + stage * Cfg::kStage;
          if (!early) ptx::mbar_expect_tx(&full_bar[stage], Cfg::kStage);
#pragma unroll
          for (int l = 0; l < NL; ++l) {
            ptx::tma_load_5d(&p.a[amap + s], &full_bar[stage], st + l * kATile, c * kChunk, xx, yy, tc.n0, l);
            if (!early)
              ptx::tma_load_3d(&p.w, &full_bar[stage], st + NL * kATile + l * Cfg::kBTile, kb * kChunk, tc.nt * BN,
                               l * p.n_phases + tc.z);
          }
        }
        __syncwarp();
        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
      }
      if (lane == 0) trace_tile(p, lt, 7);
    }
  } else if (warp >= 4) {
    // ===================================================================== consumers (warpgroups 1, 2)
    ptx::pdl_wait();   // residual reads, output / split-K partial writes must not overtake the previous kernel
    const int cw = (warp >> 2) - 1;                         // rows [64cw, 64cw + 64) of every tile
    const bool wg_leader = (threadIdx.x & 127) == 0;
    int stage = 0;
    uint32_t phase = 0;
    int lt = 0;
    for (int t = t0; t < p.total_tiles; t += tstep, ++lt) {
      const TileCoord tc = decode_tile(p, t);
      const int kb0 = tc.split * p.split_len;
      const int kb1 = (kb0 + p.split_len < num_kb) ? kb0 + p.split_len : num_kb;
      if (threadIdx.x == 128) trace_tile(p, lt, 0);
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.0f;
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        ptx::mbar_wait(&full_bar[stage], phase);
        if (threadIdx.x == 128 && kb == kb0) trace_tile(p, lt, 1);
        ptx::wgmma_fence();
        const uint32_t a0 = ptx::smem_u32(smem + stage * Cfg::kStage) + cw * 64 * 128;
        const uint32_t b0 = ptx::smem_u32(smem + stage * Cfg::kStage) + NL * kATile;
        const uint64_t a_hi = ptx::gmma_desc_sw128(a0);
        const uint64_t b_hi = ptx::gmma_desc_sw128(b0);
#pragma unroll
        for (int k = 0; k < kChunk / 16; ++k) {
          const uint32_t accum = (kb > kb0 || k > 0) ? 1u : 0u;
          // +32 bytes along K inside the 128-byte swizzle row = +2 in descriptor address units
          ptx::wgmma_m64k16<BN, NL == 2>(acc, a_hi + 2 * k, b_hi + 2 * k, accum);
          if constexpr (NL == 2) {
            const uint64_t a_lo = ptx::gmma_desc_sw128(a0 + kATile);
            const uint64_t b_lo = ptx::gmma_desc_sw128(b0 + Cfg::kBTile);
            ptx::wgmma_m64k16<BN, true>(acc, a_hi + 2 * k, b_lo + 2 * k, 1u);
            ptx::wgmma_m64k16<BN, true>(acc, a_lo + 2 * k, b_hi + 2 * k, 1u);
          }
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<1>();                                // the previous stage's MMAs have retired: hand it back
        if (prev >= 0 && wg_leader) release_stage<1>(&empty_bar[prev]);
        prev = stage;
        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
      }
      ptx::wgmma_wait<0>();
      if (prev >= 0 && wg_leader) release_stage<1>(&empty_bar[prev]);
      if (threadIdx.x == 128) trace_tile(p, lt, 2);
      epilogue_regs<BN, NL, false>(p, acc, tc, t, 64 * cw, nullptr, 0);
      if (threadIdx.x == 128) trace_tile(p, lt, 3);
    }
  }
  if (threadIdx.x == 0) trace_time(p, true);
}


// ====================================================================================================
// Patch mode.  The per-tap kernel above re-loads a 16 KB A tile for every tap, i.e. reads the layer input 9x from L2.
// Here ONE halo patch {64 ch, TW+halo, TH+halo} is loaded per (tile, source, 64-channel chunk) and all taps are
// addressed inside it: with TW = 8 an 8-row core-matrix group of the wgmma A operand is one image row of the patch, so
// the shifted A tile of tap (dx,dy) is the same swizzled buffer described by
//   start = patch + ((dy-dy0)*PW + (dx-dx0)) * 128 B,   stride between 8-row groups (SBO) = PW * 128 B,
// and tile rows 64..127 (the second m64 MMA) start 8 image rows further down.
// The swizzle phase of a row is a function of its absolute smem address for both TMA and the tensor core, so rows that
// TMA wrote are read back consistently at any 128-byte-aligned start (descriptor base offset 0).
// A and B move through separate mbarrier rings: an A patch is consumed by n_taps B tiles.
// The consumers ping-pong: warpgroup 1 owns the CTA's even local tiles and warpgroup 2 the odd ones, all 128 rows of
// each (two m64nBN accumulators), so one warpgroup runs its epilogue while the other issues the next tile's MMAs.
// ====================================================================================================
constexpr int kPatchSlot = 23 * 1024;           // >= 10*18*128 = 23040 bytes
constexpr int kPatchStride = 23 * 1024;         // distance between patch buffers (1024-byte aligned)

// Register split of the patch kernel (setmaxnreg): the launch gives every thread 168 registers (384 threads, one CTA per
// SM); the producer warpgroup gives most of its share to the consumers, which hold 2 x BN/2 accumulator floats each.
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;
static_assert(128 * kProducerRegs + 256 * kConsumerRegs <= 65536, "register file of one SM");

template <int BN, int NL, bool TAIL>
struct PatchCfg {
  using Aux = AuxCfg<TAIL>;
  static constexpr int kBTile = BN * 128;
  // taps per B stage: each stage costs one barrier round trip, so a stage must carry enough tensor work: 2 taps for
  // N=128 bf16, 2-3 for N=64, all 9 for the tail.
  static constexpr int kTPS = TAIL ? 9 : (BN >= 128 ? (NL == 1 ? 2 : 1) : (NL == 1 ? 3 : 2));
  static constexpr int kAStage = NL * kPatchStride;
  static constexpr int kBStage = NL * kTPS * kBTile;
  // Two A patches are enough (the next one is requested a full chunk ahead); everything else goes to B stages.
  static constexpr int kAStages = 2;
  static constexpr int kAvail = kSmemBudget - 1024 - Aux::kBytes - kAStages * kAStage;
  static constexpr int kBStagesRaw = kAvail / kBStage;
  static constexpr int kBStages = kBStagesRaw > 12 ? 12 : kBStagesRaw;
  static constexpr int kSmemBytes = 1024 + kAStages * kAStage + kBStages * kBStage + Aux::kBytes;
  static_assert(kBStages >= 2, "B ring needs at least two stages");
  static_assert(BN == 16 || BN == 64 || BN == 128, "instantiated N tiles");
};

// CL = cluster size (1 or 2).  With CL = 2 the two CTAs of a cluster work on neighbouring M tiles of the same N tile and
// phase, so they consume identical B stages: each CTA fetches half the rows of every weight tile and multicasts them
// to both (cp.async.bulk.tensor ... .multicast::cluster), halving the L2->SM weight traffic.  A stage is refilled only
// after both CTAs' consumers released it (remote mbarrier arrives).
template <int BN, int NL, bool TAIL, int CL>
__global__ void __launch_bounds__(kThreads, 1) conv_patch_kernel(const __grid_constant__ ConvParams p) {
  using Cfg = PatchCfg<BN, NL, TAIL>;
  const int t0 = static_cast<int>(blockIdx.x), tstep = static_cast<int>(gridDim.x);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_ring = smem;
  uint8_t* b_ring = a_ring + Cfg::kAStages * Cfg::kAStage;
  uint8_t* aux = b_ring + Cfg::kBStages * Cfg::kBStage;
  uint64_t* afull_bar = reinterpret_cast<uint64_t*>(aux);  // [kAStages]
  uint64_t* aempty_bar = afull_bar + Cfg::kAStages;         // [kAStages]
  uint64_t* bfull_bar = aempty_bar + Cfg::kAStages;         // [kBStages]
  uint64_t* bempty_bar = bfull_bar + Cfg::kBStages;         // [kBStages]
  uint64_t* turn_bar = bempty_bar + Cfg::kBStages;          // [2]: consumer warpgroup w has issued every MMA of a tile
  float* tail_stg = reinterpret_cast<float*>(aux + kBarBytes);

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);   // provably warp-uniform
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) { trace_stamp(p, 0); trace_time(p, false); }

  if (warp == 0 && lane == 0) {
    for (int i = 0; i < 4; ++i) ptx::prefetch_tmap(&p.a[i]);
    ptx::prefetch_tmap(&p.w);
    // every stage is consumed by the one warpgroup that owns its tile (in each CTA of the cluster for B)
    for (int i = 0; i < Cfg::kAStages; ++i) { ptx::mbar_init(&afull_bar[i], 1); ptx::mbar_init(&aempty_bar[i], 1); }
    for (int i = 0; i < Cfg::kBStages; ++i) { ptx::mbar_init(&bfull_bar[i], 1); ptx::mbar_init(&bempty_bar[i], CL); }
    for (int i = 0; i < 2; ++i) ptx::mbar_init(&turn_bar[i], 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  if (CL > 1) ptx::cluster_sync();     // the peer's barriers are initialised before it is sent multicast data or remote arrives
  const uint32_t crank = (CL > 1) ? ptx::cluster_ctarank() : 0u;
  constexpr uint16_t kMask = static_cast<uint16_t>((1u << CL) - 1u);
  ptx::pdl_launch_dependents();   // the next kernel may start its prologue; it waits (pdl_wait) before touching our output
  if (threadIdx.x == 0) trace_stamp(p, 1);

  int kb_per_tap = 0;
  for (int s = 0; s < p.n_src; ++s) kb_per_tap += p.chunks[s];   // = (source, chunk) items per tile
  const int patch_bytes = p.patch_w * p.patch_h * 128;
  const int n_groups = (p.n_taps + Cfg::kTPS - 1) / Cfg::kTPS;

  if (warp < 4) {
    ptx::setmaxnreg_dec<kProducerRegs>();   // the whole warpgroup; warps 1-3 have no further work
    if (warp == 0) {
      // ===================================================================== TMA producer
      // Flat sequence of items (tile, concat-chunk ci).  The A patch of item j+1 is issued in the middle of item
      // j's B tiles so that it is in flight while the consumers still work on item j.
      ptx::pdl_wait();                // activations are written by the previous kernel
      int ia = 0, ib = 0;
      uint32_t pha = 0, phb = 0;
      int a_tile = t0, a_ci = -1;            // cursor of the next A patch to issue (-1: take the tile's first item)
      auto issue_a = [&]() {
        if (a_tile >= p.total_tiles) return;
        const TileCoord tc = decode_tile(p, a_tile);
        const int ci0 = tc.split * p.split_len;
        const int ci1 = (ci0 + p.split_len < kb_per_tap) ? ci0 + p.split_len : kb_per_tap;
        if (a_ci < 0) a_ci = ci0;
        const int s = (a_ci < p.chunks[0]) ? 0 : 1;
        const int c = (s == 0) ? a_ci : a_ci - p.chunks[0];
        ptx::mbar_wait(&aempty_bar[ia], pha ^ 1);
        if (ptx::elect_one()) {
          ptx::mbar_expect_tx(&afull_bar[ia], NL * patch_bytes);
#pragma unroll
          for (int l = 0; l < NL; ++l)
            ptx::tma_load_5d(&p.a[s], &afull_bar[ia], a_ring + ia * Cfg::kAStage + l * kPatchStride, c * kChunk,
                             tc.x0 + p.patch_dx0[tc.z], tc.y0 + p.patch_dy0[tc.z], tc.n0, l);
        }
        __syncwarp();
        if (++ia == Cfg::kAStages) { ia = 0; pha ^= 1; }
        if (++a_ci == ci1) { a_ci = -1; a_tile += tstep; }
      };
      issue_a();
      const int a_after_group = (n_groups > 1) ? 1 : 0;
      int lt = 0;
      for (int t = t0; t < p.total_tiles; t += tstep, ++lt) {
        const TileCoord tc = decode_tile(p, t);
        const int ci0 = tc.split * p.split_len;
        const int ci1 = (ci0 + p.split_len < kb_per_tap) ? ci0 + p.split_len : kb_per_tap;
        if (lane == 0) trace_tile(p, lt, 6);
        for (int ci = ci0; ci < ci1; ++ci) {
          for (int g = 0; g < n_groups; ++g) {
            ptx::mbar_wait(&bempty_bar[ib], phb ^ 1);
            if (ptx::elect_one()) {
              uint8_t* st = b_ring + ib * Cfg::kBStage;
              if constexpr (CL == 1 && NL == 1) {
                ptx::mbar_expect_tx(&bfull_bar[ib], Cfg::kBStage);
                // one box = kTPS taps x BN rows x 64 channels (taps beyond n_taps are zero-filled)
                ptx::tma_load_4d(&p.w, &bfull_bar[ib], st, ci * kChunk, tc.nt * BN, g * Cfg::kTPS, tc.z);
              } else {
                // per-tap boxes of BN/CL rows.  Stage layout [tap][limb][BN rows].  With CL = 2 this CTA fetches rows
                // [crank*BN/CL, +BN/CL) of every tile and multicasts them to the whole cluster.
                const int tap0 = g * Cfg::kTPS;
                const int ntap = (tap0 + Cfg::kTPS < p.n_taps) ? Cfg::kTPS : p.n_taps - tap0;
                ptx::mbar_expect_tx(&bfull_bar[ib], NL * ntap * Cfg::kBTile);
                constexpr int kRows = BN / CL;
                for (int ti = 0; ti < ntap; ++ti)
#pragma unroll
                  for (int l = 0; l < NL; ++l) {
                    uint8_t* dst = st + (ti * NL + l) * Cfg::kBTile + crank * kRows * 128;
                    if constexpr (CL == 1)
                      ptx::tma_load_4d(&p.w, &bfull_bar[ib], dst, ci * kChunk, tc.nt * BN, tap0 + ti, l * p.n_phases + tc.z);
                    else
                      ptx::tma_load_4d_mc(&p.w, &bfull_bar[ib], dst, ci * kChunk, tc.nt * BN + crank * kRows, tap0 + ti,
                                          l * p.n_phases + tc.z, kMask);
                  }
              }
            }
            __syncwarp();
            if (++ib == Cfg::kBStages) { ib = 0; phb ^= 1; }
            if (g == a_after_group) issue_a();
          }
        }
        if (lane == 0) trace_tile(p, lt, 7);
      }
    }
  } else {
    ptx::setmaxnreg_inc<kConsumerRegs>();
    // ===================================================================== consumers (warpgroups 1, 2)
    // Ping-pong: warpgroup w owns the local tiles lt with lt % 2 == w, all 128 rows (acc[0]: rows 0-63, acc[1]: rows
    // 64-127, read 8 image rows further down the patch).  Every accumulator element sees the same operands in the same
    // K order as one m64 half of a tile split across both warpgroups would.  A ring stage is consumed by the warpgroup
    // that owns its tile; the other one moves its cursors past the tile's stages.
    // MMA issue alternates by tile: tile lt > 0 starts once the other warpgroup has issued every MMA of tile lt-1
    // (turn_bar), so the tensor pipe finishes one tile before it starts the next and the owner's epilogue runs under the
    // next tile's MMAs.  This cannot deadlock: issuing tile lt-1 needs only the stages of tile lt-1, which the producer
    // fills in tile order into slots freed by tiles <= lt-2, and the waiting warpgroup released every stage of its own
    // tile lt-2 before its epilogue.  Each wait depends on an event of an earlier tile only.
    ptx::pdl_wait();   // residual reads, output / split-K partial writes must not overtake the previous kernel
    const int wg = (warp >> 2) - 1;
    const bool wg_leader = (threadIdx.x & 127) == 0;
    int ia = 0, ib = 0;
    uint32_t pha = 0, phb = 0;
    const uint32_t sbo = static_cast<uint32_t>(p.patch_w) * 128u;
    const uint32_t row_off = static_cast<uint32_t>(8 * p.patch_w) * 128u;   // tile rows 64..127: 8 image rows down
    float* stg = tail_stg + wg * kTileM * kTailStride;                       // this warpgroup's tail staging (128 rows)
    int lt = 0;
    for (int t = t0; t < p.total_tiles; t += tstep, ++lt) {
      const TileCoord tc = decode_tile(p, t);
      const int ci0 = tc.split * p.split_len;
      const int ci1 = (ci0 + p.split_len < kb_per_tap) ? ci0 + p.split_len : kb_per_tap;
      if ((lt & 1) != wg) {
        // the other warpgroup's tile: (ci1 - ci0) A patches and n_groups B stages per patch
        ia += ci1 - ci0;
        pha ^= static_cast<uint32_t>(ia / Cfg::kAStages) & 1u;
        ia %= Cfg::kAStages;
        ib += (ci1 - ci0) * n_groups;
        phb ^= static_cast<uint32_t>(ib / Cfg::kBStages) & 1u;
        ib %= Cfg::kBStages;
        continue;
      }
      if (lt > 0) ptx::mbar_wait(&turn_bar[wg ^ 1], static_cast<uint32_t>((lt - 1) >> 1) & 1u);
      if (wg_leader) trace_tile(p, lt, 0);
      float acc[2][BN / 2];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[h][i] = 0.0f;
      // the stage consumed one step earlier is released once the MMAs that read it have retired (wgmma.wait_group 1)
      int prev_b = -1, prev_a = -1;
      for (int ci = ci0; ci < ci1; ++ci) {
        ptx::mbar_wait(&afull_bar[ia], pha);
        const uint32_t a0 = ptx::smem_u32(a_ring + ia * Cfg::kAStage);
        for (int g = 0; g < n_groups; ++g) {
          ptx::mbar_wait(&bfull_bar[ib], phb);
          if (wg_leader && ci == ci0 && g == 0) trace_tile(p, lt, 1);
          ptx::wgmma_fence();
          const int tap0 = g * Cfg::kTPS;
          const uint32_t b0 = ptx::smem_u32(b_ring + ib * Cfg::kBStage);
#pragma unroll
          for (int i = 0; i < Cfg::kTPS; ++i) {
            const int tap = tap0 + i;
            if (i == 0 || tap < p.n_taps) {                     // the last group may be short (never empty)
              const uint32_t a_hi_addr = a0 + static_cast<uint32_t>(p.tap_row[tc.z][tap]) * 128u;
              const uint32_t b_hi_addr = b0 + static_cast<uint32_t>(i) * (NL * Cfg::kBTile);
              const uint64_t b_hi = ptx::gmma_desc_sw128(b_hi_addr);
              const uint64_t b_lo = ptx::gmma_desc_sw128(b_hi_addr + Cfg::kBTile);   // PARITY only
#pragma unroll
              for (int k = 0; k < kChunk / 16; ++k) {
                const uint32_t accum = (ci > ci0 || tap > 0 || k > 0) ? 1u : 0u;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  const uint64_t a_hi = ptx::gmma_desc_sw128(a_hi_addr + h * row_off, sbo);
                  ptx::wgmma_m64k16<BN, NL == 2>(acc[h], a_hi + 2 * k, b_hi + 2 * k, accum);
                  if constexpr (NL == 2) {
                    const uint64_t a_lo = ptx::gmma_desc_sw128(a_hi_addr + h * row_off + kPatchStride, sbo);
                    ptx::wgmma_m64k16<BN, true>(acc[h], a_hi + 2 * k, b_lo + 2 * k, 1u);
                    ptx::wgmma_m64k16<BN, true>(acc[h], a_lo + 2 * k, b_hi + 2 * k, 1u);
                  }
                }
              }
            }
          }
          ptx::wgmma_commit();
          if (ci == ci1 - 1 && g == n_groups - 1 && wg_leader) ptx::mbar_arrive(&turn_bar[wg]);   // tile fully issued
          ptx::wgmma_wait<1>();
          if (wg_leader) {
            if (prev_b >= 0) release_stage<CL>(&bempty_bar[prev_b]);
            if (prev_a >= 0) ptx::mbar_arrive(&aempty_bar[prev_a]);
          }
          prev_b = ib;
          prev_a = (g == n_groups - 1) ? ia : -1;              // the patch is free after its last group of taps
          if (++ib == Cfg::kBStages) { ib = 0; phb ^= 1; }
        }
        if (++ia == Cfg::kAStages) { ia = 0; pha ^= 1; }
      }
      ptx::wgmma_wait<0>();
      if (wg_leader) {
        if (prev_b >= 0) release_stage<CL>(&bempty_bar[prev_b]);
        if (prev_a >= 0) ptx::mbar_arrive(&aempty_bar[prev_a]);
      }
      if (wg_leader) trace_tile(p, lt, 2);
#pragma unroll
      for (int h = 0; h < 2; ++h)
        epilogue_regs<BN, NL, TAIL>(p, acc[h], tc, t, 64 * h, stg + 64 * h * kTailStride, 1 + wg);
      if (wg_leader) trace_tile(p, lt, 3);
    }
  }
  if (CL > 1) ptx::cluster_sync();     // no CTA leaves while a peer may still signal its barriers / write its smem
  if (threadIdx.x == 0) trace_time(p, true);
}

// ====================================================================================================
// Split-K finisher: out = epilogue( sum_s partial[s] ).
// Memory-bound and tiny (the layers that use split-K have at most a few hundred output pixels per image).
// ====================================================================================================
// One thread = one pixel x 4 channels.  The layers that use split-K are latency bound (a few hundred output pixels, 8-36
// splits): what matters is how many dependent trips to L2 the sum takes, so up to 16 splits are in flight per trip
// (round 1 summed 4 per trip over 8-channel groups: 6 dependent trips for 18 splits, as long as the conv itself at batch 1).
// It reads the conv launch's own parameters; the split-K layers are never the tail, so the output has Cout_pad channels.
template <int NL>
__global__ void __launch_bounds__(128) splitk_reduce_kernel(const __grid_constant__ ConvParams p) {
  ptx::pdl_wait();
  ptx::pdl_launch_dependents();
  const int bn = p.out_channels / p.n_tiles;
  const int groups = bn >> 2;
  const long long total = static_cast<long long>(p.tiles_per_split) * kTileM * groups;
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(e % groups);
    const long long r0 = e / groups;
    const int row = static_cast<int>(r0 % kTileM);
    const int tile = static_cast<int>(r0 / kTileM);
    const TileCoord tc = decode_tile(p, tile);       // split 0: tile < tiles_per_split
    int n, y, x;
    row_pixel(p, tc, row, n, y, x);
    if (n >= p.batch || y >= p.hs || x >= p.ws) continue;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const size_t split_stride = static_cast<size_t>(p.tiles_per_split) * kTileM * bn;      // floats between splits
    const float* src0 = p.partial + (static_cast<size_t>(tile) * kTileM + row) * bn + g * 4;
    int s = 0;
    for (; s + 16 <= p.n_split; s += 16) {     // sixteen independent 16-byte loads in flight
      float4 v[16];
#pragma unroll
      for (int u = 0; u < 16; ++u) v[u] = *reinterpret_cast<const float4*>(src0 + (s + u) * split_stride);
#pragma unroll
      for (int u = 0; u < 16; ++u) {           // summation order stays s = 0, 1, 2, ... (deterministic)
        acc[0] += v[u].x; acc[1] += v[u].y; acc[2] += v[u].z; acc[3] += v[u].w;
      }
    }
    for (; s + 4 <= p.n_split; s += 4) {
      float4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = *reinterpret_cast<const float4*>(src0 + (s + u) * split_stride);
#pragma unroll
      for (int u = 0; u < 4; ++u) { acc[0] += v[u].x; acc[1] += v[u].y; acc[2] += v[u].z; acc[3] += v[u].w; }
    }
    for (; s < p.n_split; ++s) {
      const float4 a = *reinterpret_cast<const float4*>(src0 + s * split_stride);
      acc[0] += a.x; acc[1] += a.y; acc[2] += a.z; acc[3] += a.w;
    }
    const int ch = tc.nt * bn + g * 4;
    __nv_bfloat16* out = out_pixel(p, tc, n, y, x) + ch;
    const float4 sc = *reinterpret_cast<const float4*>(p.scale + ch), sh = *reinterpret_cast<const float4*>(p.shift + ch);
    uint32_t rw[NL][2];                          // per limb: residual words of channels (ch, ch+1) and (ch+2, ch+3)
    if (p.has_res) {
      const size_t roff = ((static_cast<size_t>(n) * p.hs + y) * p.ws + x) * p.res_channels + ch;
#pragma unroll
      for (int l = 0; l < NL; ++l) {
        const uint2 r = *reinterpret_cast<const uint2*>(p.res_ptr + l * p.res_limb_stride + roff);
        rw[l][0] = r.x; rw[l][1] = r.y;
      }
    }
    epilogue_pair<2>(p, acc[0], acc[1], make_float2(sc.x, sc.y), make_float2(sh.x, sh.y), rw, 0, out);
    epilogue_pair<2>(p, acc[2], acc[3], make_float2(sc.z, sc.w), make_float2(sh.z, sh.w), rw, 1, out);
  }
}

}  // namespace lspg
