// C-ABI implementation of the baseline JPEG encoder (see include/lspj.h; oracle/jpeg_oracle.py restates it in numpy).
//
// Four launches per call, all on the caller's stream:
//   1. lspj_block_kernel, one thread per 8x8 block of the scan: colour conversion (and the 2x2 chroma downsampling) of
//      its pixels, the islow FDCT, quantisation; stores the 64 zigzagged coefficients and the block's AC bit count.
//   2. lspj_offsets_kernel, one CTA per frame: adds each block's DC bits (the DC prediction needs only the previous
//      block's quantised DC), an exclusive scan of the bit counts gives each block's first bit, and the frame's bit
//      buffer is zeroed up to its total.
//   3. lspj_pack_kernel, one thread per block: Huffman-codes the block at its offset, MSB first in 32-bit words.  A
//      word can straddle two blocks, so every word is written with atomicOr (order-free, so the bytes do not vary).
//   4. lspj_stuff_kernel, one CTA per frame: copies the scan bytes (the last one padded with 1 bits) behind the header
//      with a 0x00 after every 0xFF, 16 bytes per thread per round with a block scan of the output lengths, then writes
//      the header, EOI and the file's size.
// Integer arithmetic throughout: the bytes are the same from run to run and equal libjpeg-turbo's.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>

#include "../../include/lspj.h"
#include "bitstream.cuh"
#include "capi.cuh"

using bitstream::block_exclusive_scan;
using bitstream::BitWriter;
using bitstream::Sum;
using capi::align256;
using capi::DeviceGuard;

namespace {

struct Lspj;
constexpr auto fail = capi::fail<Lspj>;

constexpr int kWorstBlockBits = 16 + 11 + 63 * (16 + 10) + 3 * 16 + 16;   // 1729, derived in lspj.h
constexpr int kMaxHeader = 640;
constexpr int kBlockThreads = 128;
constexpr int kFrameThreads = 1024;
constexpr int64_t kMaxFileBytes = int64_t(1) << 30;

// ---- the standard tables (JPEG standard Annex K; jcparam / jstdhuff) --------------------------------------------

constexpr uint8_t kLumaQuant[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,
                                    14, 13, 16, 24, 40,  57,  69,  56,  14, 17, 22, 29, 51,  87,  80,  62,
                                    18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
                                    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
constexpr uint8_t kChromaQuant[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99,
                                      24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
                                      99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                                      99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
// zigzag position -> natural index (jpeg_natural_order); called with constant k only, so it folds away in device code
__host__ __device__ constexpr int zigzag(int k) {
  constexpr uint8_t t[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                             41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                             30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
  return t[k];
}

struct HuffSpec {
  uint8_t bits[16];
  uint8_t vals[162];
};
// DC luma, AC luma, DC chroma, AC chroma: jcmarker's DHT order
constexpr HuffSpec kHuffSpec[4] = {
    {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0}, {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11}},
    {{0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d},
     {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
      0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
      0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,
      0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65,
      0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
      0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
      0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
      0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea,
      0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}},
    {{0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}, {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11}},
    {{0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77},
     {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
      0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16,
      0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39,
      0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
      0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86,
      0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
      0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8,
      0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9,
      0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}}};

// jpeg_make_c_derived_tbl: entry (size << 16) | code per symbol, size 0 for symbols without a code
struct HuffCodes {
  uint32_t e[4][256];
};

constexpr HuffCodes make_codes() {
  HuffCodes t{};
  for (int i = 0; i < 4; ++i) {
    uint32_t code = 0;
    int k = 0;
    for (int len = 1; len <= 16; ++len) {
      for (int j = 0; j < kHuffSpec[i].bits[len - 1]; ++j, ++k, ++code)
        t.e[i][kHuffSpec[i].vals[k]] = (static_cast<uint32_t>(len) << 16) | code;
      code <<= 1;
    }
  }
  return t;
}

__constant__ HuffCodes kCodes = make_codes();

// ---- launch parameters --------------------------------------------------------------------------------------------

struct FrameLayout {            // one frame's share of the workspace
  size_t coef, offs, bits, bytes;
};

struct Params {
  const uint8_t* images;
  int64_t image_stride;         // bytes per input frame
  uint8_t* out;
  int64_t out_stride;
  int32_t* sizes;
  uint8_t* ws;
  FrameLayout lay;
  int width, comps, nblk, header_len;
  uint16_t qdiv[2][64];         // 8 * table, zigzag order
  uint8_t header[kMaxHeader];
};

__device__ __forceinline__ int16_t* frame_coef(const Params& p, int f) {
  return reinterpret_cast<int16_t*>(p.ws + f * p.lay.bytes + p.lay.coef);
}
__device__ __forceinline__ uint32_t* frame_offs(const Params& p, int f) {
  return reinterpret_cast<uint32_t*>(p.ws + f * p.lay.bytes + p.lay.offs);
}
__device__ __forceinline__ uint32_t* frame_bits(const Params& p, int f) {
  return reinterpret_cast<uint32_t*>(p.ws + f * p.lay.bytes + p.lay.bits);
}

__device__ __forceinline__ int nbits(int v) { return v == 0 ? 0 : 32 - __clz(v < 0 ? -v : v); }

// The scan's previous block of the same component (DC prediction), or -1.  Colour: MCU m holds blocks 6m..6m+5.
__device__ __forceinline__ int prev_block(int b, int comps) {
  if (comps == 1) return b - 1;
  const int j = b % 6;
  if (j >= 4) return b - 6;                                 // Cb, Cr: the same slot of the previous MCU
  return j > 0 ? b - 1 : b - 3;                             // Y0 follows the previous MCU's Y3 (b - 6 + 3)
}

// One jfdctint pass over 8 values v[0], v[s], ..., v[7 s].
template <bool kRows>
__device__ __forceinline__ void fdct_pass(int* v, int s) {
  constexpr int kConst = 13, kPass1 = 2, kShift = kRows ? kConst - kPass1 : kConst + kPass1;
  const int t0 = v[0] + v[7 * s], t7 = v[0] - v[7 * s], t1 = v[s] + v[6 * s], t6 = v[s] - v[6 * s];
  const int t2 = v[2 * s] + v[5 * s], t5 = v[2 * s] - v[5 * s], t3 = v[3 * s] + v[4 * s], t4 = v[3 * s] - v[4 * s];
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  if (kRows) {
    v[0] = (t10 + t11) * (1 << kPass1);
    v[4 * s] = (t10 - t11) * (1 << kPass1);
  } else {
    v[0] = (t10 + t11 + (1 << (kPass1 - 1))) >> kPass1;
    v[4 * s] = (t10 - t11 + (1 << (kPass1 - 1))) >> kPass1;
  }
  constexpr int kRound = 1 << (kShift - 1);
  int z1 = (t12 + t13) * 4433;
  v[2 * s] = (z1 + t13 * 6270 + kRound) >> kShift;
  v[6 * s] = (z1 - t12 * 15137 + kRound) >> kShift;
  z1 = t4 + t7;
  int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
  const int z5 = (z3 + z4) * 9633;
  const int a4 = t4 * 2446, a5 = t5 * 16819, a6 = t6 * 25172, a7 = t7 * 12299;
  z1 *= -7373;
  z2 *= -20995;
  z3 = z3 * -16069 + z5;
  z4 = z4 * -3196 + z5;
  v[7 * s] = (a4 + z1 + z3 + kRound) >> kShift;
  v[5 * s] = (a5 + z2 + z4 + kRound) >> kShift;
  v[3 * s] = (a6 + z2 + z3 + kRound) >> kShift;
  v[s] = (a7 + z1 + z4 + kRound) >> kShift;
}

__device__ __forceinline__ int luma(int r, int g, int b) { return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16; }

__device__ __forceinline__ void load_huff(uint32_t* s) {
  for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) s[i] = kCodes.e[i >> 8][i & 255];
}

// ---- 1. colour, downsampling, FDCT, quantisation -------------------------------------------------------------------

__global__ void __launch_bounds__(kBlockThreads) lspj_block_kernel(const Params p) {
  __shared__ uint32_t huff[4 * 256];
  load_huff(huff);
  __syncthreads();
  const int f = blockIdx.y, b = blockIdx.x * kBlockThreads + threadIdx.x;
  if (b >= p.nblk) return;
  const uint8_t* img = p.images + f * p.image_stride;
  int v[64];
  int comp;
  if (p.comps == 1) {
    comp = 0;
    const int bw = p.width >> 3, x = (b % bw) * 8, y = (b / bw) * 8;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const uint2 w = __ldg(reinterpret_cast<const uint2*>(img + static_cast<int64_t>(y + r) * p.width + x));
#pragma unroll
      for (int c = 0; c < 8; ++c) v[r * 8 + c] = static_cast<int>(((c < 4 ? w.x : w.y) >> (8 * (c & 3))) & 255) - 128;
    }
  } else {
    const int mw = p.width >> 4, m = b / 6, j = b - m * 6;
    const int x0 = (m % mw) * 16, y0 = (m / mw) * 16;
    comp = j < 4 ? 0 : j - 3;
    if (comp == 0) {
      const int x = x0 + 8 * (j & 1), y = y0 + 8 * (j >> 1);
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const uint2* row = reinterpret_cast<const uint2*>(img + (static_cast<int64_t>(y + r) * p.width + x) * 3);
        const uint2 a = __ldg(row), bb = __ldg(row + 1), c2 = __ldg(row + 2);
        const uint32_t w[6] = {a.x, a.y, bb.x, bb.y, c2.x, c2.y};
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const int rr = (w[(3 * c) >> 2] >> (8 * ((3 * c) & 3))) & 255;
          const int gg = (w[(3 * c + 1) >> 2] >> (8 * ((3 * c + 1) & 3))) & 255;
          const int bl = (w[(3 * c + 2) >> 2] >> (8 * ((3 * c + 2) & 3))) & 255;
          v[r * 8 + c] = luma(rr, gg, bl) - 128;
        }
      }
    } else {
      // Cb = (-11059 r - 21709 g + 32768 b + (128 << 16) + 32767) >> 16, Cr = (32768 r - 27439 g - 5329 b + ...) >> 16
      const int kr = comp == 1 ? -11059 : 32768, kg = comp == 1 ? -21709 : -27439, kb = comp == 1 ? 32768 : -5329;
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        int sum[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) sum[c] = (c & 1) ? 2 : 1;              // h2v2_downsample's alternating bias
#pragma unroll
        for (int dy = 0; dy < 2; ++dy) {
          const uint4* row = reinterpret_cast<const uint4*>(img + (static_cast<int64_t>(y0 + 2 * r + dy) * p.width + x0) * 3);
          const uint4 a = __ldg(row), bb = __ldg(row + 1), c2 = __ldg(row + 2);
          const uint32_t w[12] = {a.x, a.y, a.z, a.w, bb.x, bb.y, bb.z, bb.w, c2.x, c2.y, c2.z, c2.w};
#pragma unroll
          for (int px = 0; px < 16; ++px) {
            const int rr = (w[(3 * px) >> 2] >> (8 * ((3 * px) & 3))) & 255;
            const int gg = (w[(3 * px + 1) >> 2] >> (8 * ((3 * px + 1) & 3))) & 255;
            const int bl = (w[(3 * px + 2) >> 2] >> (8 * ((3 * px + 2) & 3))) & 255;
            sum[px >> 1] += (kr * rr + kg * gg + kb * bl + (128 << 16) + 32767) >> 16;
          }
        }
#pragma unroll
        for (int c = 0; c < 8; ++c) v[r * 8 + c] = (sum[c] >> 2) - 128;
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 8; ++r) fdct_pass<true>(v + 8 * r, 1);
#pragma unroll
  for (int c = 0; c < 8; ++c) fdct_pass<false>(v + c, 8);
  // quantise in zigzag order, store, and count the AC bits
  const uint32_t* ac = huff + (comp > 0 ? 3 : 1) * 256;
  uint32_t packed[32];
  int bits = 0, run = 0;
#pragma unroll
  for (int k = 0; k < 64; ++k) {
    const int x = v[zigzag(k)], d = comp > 0 ? p.qdiv[1][k] : p.qdiv[0][k];
    const int a = (x < 0 ? -x : x) + (d >> 1);
    const int q = x < 0 ? -(a / d) : a / d;
    if (k & 1) packed[k >> 1] |= static_cast<uint32_t>(q) << 16;
    else packed[k >> 1] = static_cast<uint32_t>(q) & 0xffffu;
    if (k > 0) {
      if (q == 0) {
        ++run;
      } else {
        bits += (run >> 4) * (ac[0xf0] >> 16);
        run &= 15;
        const int n = nbits(q);
        bits += (ac[(run << 4) + n] >> 16) + n;
        run = 0;
      }
    }
  }
  if (run > 0) bits += ac[0] >> 16;
  uint4* dst = reinterpret_cast<uint4*>(frame_coef(p, f) + static_cast<int64_t>(b) * 64);
#pragma unroll
  for (int i = 0; i < 8; ++i) dst[i] = make_uint4(packed[4 * i], packed[4 * i + 1], packed[4 * i + 2], packed[4 * i + 3]);
  frame_offs(p, f)[b] = bits;
}

// ---- 2. DC bits, bit offsets, zeroed bit buffer ---------------------------------------------------------------------

__device__ __forceinline__ uint32_t dc_bits(const int16_t* coef, int b, int comps) {
  const int pb = prev_block(b, comps);
  const int diff = coef[static_cast<int64_t>(b) * 64] - (pb >= 0 ? coef[static_cast<int64_t>(pb) * 64] : 0);
  const int n = nbits(diff);
  const bool chroma = comps == 3 && b % 6 >= 4;
  return (kCodes.e[chroma ? 2 : 0][n] >> 16) + n;
}

__global__ void __launch_bounds__(kFrameThreads) lspj_offsets_kernel(const Params p) {
  const int f = blockIdx.x;
  const int16_t* coef = frame_coef(p, f);
  uint32_t* offs = frame_offs(p, f);
  const uint32_t total = bitstream::counts_to_offsets(offs, p.nblk, 0u, [&](int b) { return dc_bits(coef, b, p.comps); });
  uint32_t* buf = frame_bits(p, f);
  const uint32_t words = (total + 31) / 32;
  for (uint32_t i = threadIdx.x; i < words; i += kFrameThreads) buf[i] = 0;
}

// ---- 3. Huffman coding ----------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kBlockThreads) lspj_pack_kernel(const Params p) {
  __shared__ uint32_t huff[4 * 256];
  load_huff(huff);
  __syncthreads();
  const int f = blockIdx.y, b = blockIdx.x * kBlockThreads + threadIdx.x;
  if (b >= p.nblk) return;
  const int16_t* coef = frame_coef(p, f);
  const uint32_t off = frame_offs(p, f)[b];
  const bool chroma = p.comps == 3 && b % 6 >= 4;
  const uint32_t* dc = huff + (chroma ? 2 : 0) * 256;
  const uint32_t* ac = huff + (chroma ? 3 : 1) * 256;
  const uint4* src = reinterpret_cast<const uint4*>(coef + static_cast<int64_t>(b) * 64);
  const int pb = prev_block(b, p.comps);
  BitWriter w(frame_bits(p, f), off);
  {
    const int diff = coef[static_cast<int64_t>(b) * 64] - (pb >= 0 ? coef[static_cast<int64_t>(pb) * 64] : 0);
    const int n = nbits(diff);
    const uint32_t e = dc[n];
    w.put(e & 0xffffu, e >> 16);
    if (n) w.put(static_cast<uint32_t>(diff < 0 ? diff - 1 : diff) & ((1u << n) - 1), n);
  }
  int run = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint4 q4 = src[i];
    const uint32_t words[4] = {q4.x, q4.y, q4.z, q4.w};
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (i == 0 && k == 0) continue;                       // the DC
      const int q = static_cast<int16_t>(words[k >> 1] >> (16 * (k & 1)));
      if (q == 0) {
        ++run;
        continue;
      }
      for (; run > 15; run -= 16) w.put(ac[0xf0] & 0xffffu, ac[0xf0] >> 16);
      const int n = nbits(q);
      const uint32_t e = ac[(run << 4) + n];
      w.put(((e & 0xffffu) << n) | (static_cast<uint32_t>(q < 0 ? q - 1 : q) & ((1u << n) - 1)), (e >> 16) + n);
      run = 0;
    }
  }
  if (run > 0) w.put(ac[0] & 0xffffu, ac[0] >> 16);
  w.flush();
}

// ---- 4. byte stuffing, header, EOI ------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kFrameThreads) lspj_stuff_kernel(const Params p) {
  const int f = blockIdx.x;
  const uint32_t total = frame_offs(p, f)[p.nblk];
  const uint32_t nbytes = (total + 7) / 8;
  const uint32_t pad = (total & 7) ? (1u << (8 - (total & 7))) - 1 : 0;   // 1 bits after the last code
  const uint4* src = reinterpret_cast<const uint4*>(frame_bits(p, f));
  uint8_t* file = p.out + f * p.out_stride;
  uint8_t* dst = file + p.header_len;
  for (int i = threadIdx.x; i < p.header_len; i += kFrameThreads) file[i] = p.header[i];
  uint32_t base = 0;
  for (uint32_t r0 = 0; r0 < nbytes; r0 += 16 * kFrameThreads) {
    const uint32_t at = r0 + 16 * threadIdx.x;
    uint8_t bytes[16];
    uint32_t count = 0;
    if (at < nbytes) {
      const uint4 q = src[at >> 4];
      const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        uint32_t byte = (w[i >> 2] >> (24 - 8 * (i & 3))) & 255;
        if (at + i == nbytes - 1) byte |= pad;
        bytes[i] = static_cast<uint8_t>(byte);
        if (at + i < nbytes) count += 1 + (byte == 255);
      }
    }
    uint32_t round_total;
    uint32_t o = base + block_exclusive_scan<Sum>(count, &round_total);
    if (at < nbytes) {
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        if (at + i < nbytes) {
          dst[o++] = bytes[i];
          if (bytes[i] == 255) dst[o++] = 0;
        }
      }
    }
    base += round_total;
  }
  if (threadIdx.x == 0) {
    dst[base] = 0xff;
    dst[base + 1] = 0xd9;
    p.sizes[f] = static_cast<int32_t>(p.header_len + base + 2);
  }
}

// ---- host side ------------------------------------------------------------------------------------------------------

int check_shape(int height, int width, int components) {
  if (components != 1 && components != 3) return fail(LSPG_EINVAL, "components must be 1 or 3 (got %d)", components);
  if (height < 16 || width < 16 || height > 65535 || width > 65535 || height % 16 || width % 16)
    return fail(LSPG_EINVAL, "height and width must be multiples of 16 in [16, 65535] (got %d x %d)", height, width);
  return LSPG_OK;
}

int64_t blocks_of(int height, int width, int components) {
  const int64_t luma = static_cast<int64_t>(height / 8) * (width / 8);
  return components == 1 ? luma : luma / 4 * 6;
}

int header_bytes(uint8_t* out, int height, int width, int components, int quality) {
  int n = 0;
  auto put = [&](int v) { out[n++] = static_cast<uint8_t>(v); };
  auto put16 = [&](int v) { put(v >> 8); put(v & 255); };
  const int tables = components == 3 ? 2 : 1;
  const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;
  put(0xff), put(0xd8);
  put(0xff), put(0xe0), put16(16);
  const uint8_t jfif[14] = {'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
  for (uint8_t c : jfif) put(c);
  for (int t = 0; t < tables; ++t) {
    put(0xff), put(0xdb), put16(67), put(t);
    const uint8_t* basic = t ? kChromaQuant : kLumaQuant;
    for (int k = 0; k < 64; ++k) {
      const int v = (basic[zigzag(k)] * scale + 50) / 100;
      put(v < 1 ? 1 : v > 255 ? 255 : v);
    }
  }
  put(0xff), put(0xc0), put16(8 + 3 * components), put(8), put16(height), put16(width), put(components);
  for (int c = 0; c < components; ++c) put(c + 1), put(c == 0 && components == 3 ? 0x22 : 0x11), put(c ? 1 : 0);
  for (int t = 0; t < 2 * tables; ++t) {
    const HuffSpec& s = kHuffSpec[t];
    int nv = 0;
    for (int i = 0; i < 16; ++i) nv += s.bits[i];
    put(0xff), put(0xc4), put16(2 + 1 + 16 + nv), put(((t & 1) << 4) | (t >> 1));
    for (int i = 0; i < 16; ++i) put(s.bits[i]);
    for (int i = 0; i < nv; ++i) put(s.vals[i]);
  }
  put(0xff), put(0xda), put16(6 + 2 * components), put(components);
  for (int c = 0; c < components; ++c) put(c + 1), put(c ? 0x11 : 0x00);
  put(0), put(63), put(0);
  return n;
}

int64_t max_bytes_of(int height, int width, int components) {
  uint8_t hdr[kMaxHeader];
  const int64_t scan = (blocks_of(height, width, components) * kWorstBlockBits + 7) / 8;
  return header_bytes(hdr, height, width, components, 75) + 2 * scan + 2;
}

FrameLayout layout_of(int height, int width, int components) {
  const size_t nblk = static_cast<size_t>(blocks_of(height, width, components));
  const size_t words = (nblk * kWorstBlockBits + 31) / 32 + 4;   // + 4: the stuffing kernel reads whole uint4s
  FrameLayout l;
  l.coef = 0;
  l.offs = align256(nblk * 64 * sizeof(int16_t));
  l.bits = l.offs + align256((nblk + 1) * sizeof(uint32_t));
  l.bytes = l.bits + align256(words * sizeof(uint32_t));
  return l;
}

int check_sizes(int height, int width, int components) {
  if (int rc = check_shape(height, width, components)) return rc;
  const int64_t bound = max_bytes_of(height, width, components);
  if (bound > kMaxFileBytes)
    return fail(LSPG_EINVAL, "a %d x %d frame has a worst-case file of %lld bytes, above the 2^30 this encoder supports",
                height, width, static_cast<long long>(bound));
  return LSPG_OK;
}

}  // namespace

struct lspj_ctx {
  int device = -1;
};

extern "C" {

const char* lspj_last_error(void) { return capi::last_error<Lspj>().c_str(); }

int lspj_destroy(lspj_handle h) {
  delete h;
  return LSPG_OK;
}

int lspj_create(lspj_handle* out, int device) {
  if (!out) return fail(LSPG_EINVAL, "null argument");
  *out = nullptr;
  cudaDeviceProp prop;
  if (int rc = capi::check_device<Lspj>(device, &prop)) return rc;
  lspj_ctx* h = new lspj_ctx;
  h->device = device;
  *out = h;
  return LSPG_OK;
}

int lspj_max_bytes(lspj_handle h, int height, int width, int components, size_t* bytes) {
  if (!h || !bytes) return fail(LSPG_EINVAL, "null argument");
  if (int rc = check_sizes(height, width, components)) return rc;
  *bytes = static_cast<size_t>(max_bytes_of(height, width, components));
  return LSPG_OK;
}

int lspj_workspace_bytes(lspj_handle h, int n, int height, int width, int components, size_t* bytes) {
  if (!h || !bytes) return fail(LSPG_EINVAL, "null argument");
  if (n < 0) return fail(LSPG_EINVAL, "n must be >= 0 (got %d)", n);
  if (int rc = check_sizes(height, width, components)) return rc;
  *bytes = static_cast<size_t>(n) * layout_of(height, width, components).bytes;
  return LSPG_OK;
}

int lspj_encode(lspj_handle h, const uint8_t* images, int n, int height, int width, int components, int quality,
                uint8_t* out, int64_t out_stride, int32_t* sizes, void* ws, size_t ws_bytes, void* stream) {
  if (!h) return fail(LSPG_EINVAL, "null handle");
  if (n < 0) return fail(LSPG_EINVAL, "n must be >= 0 (got %d)", n);
  if (quality < 1 || quality > 100) return fail(LSPG_EINVAL, "quality must be in [1, 100] (got %d)", quality);
  if (int rc = check_sizes(height, width, components)) return rc;
  const int64_t bound = max_bytes_of(height, width, components);
  if (out_stride < bound)
    return fail(LSPG_EINVAL, "out_stride must be at least lspj_max_bytes = %lld (got %lld)", static_cast<long long>(bound),
                static_cast<long long>(out_stride));
  const FrameLayout lay = layout_of(height, width, components);
  if (ws_bytes < static_cast<size_t>(n) * lay.bytes)
    return fail(LSPG_EINVAL, "workspace of %zu bytes is smaller than lspj_workspace_bytes = %zu", ws_bytes,
                static_cast<size_t>(n) * lay.bytes);
  if (n > 0 && (!images || !out || !sizes || !ws)) return fail(LSPG_EINVAL, "null buffer");
  if (reinterpret_cast<uintptr_t>(images) % 16 || reinterpret_cast<uintptr_t>(ws) % 256)
    return fail(LSPG_EINVAL, "images must be 16-byte and ws 256-byte aligned");
  if (int rc = capi::require_device<Lspj>(h->device, "lspj_encode")) return rc;
  if (n == 0) return LSPG_OK;
  Params p;
  std::memset(&p, 0, sizeof(p));
  p.image_stride = static_cast<int64_t>(height) * width * components;
  p.out_stride = out_stride;
  p.lay = lay;
  p.width = width;
  p.comps = components;
  p.nblk = static_cast<int>(blocks_of(height, width, components));
  p.header_len = header_bytes(p.header, height, width, components, quality);
  const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;
  for (int t = 0; t < 2; ++t)
    for (int k = 0; k < 64; ++k) {
      const int v = ((t ? kChromaQuant : kLumaQuant)[zigzag(k)] * scale + 50) / 100;
      p.qdiv[t][k] = static_cast<uint16_t>(8 * (v < 1 ? 1 : v > 255 ? 255 : v));
    }
  DeviceGuard g(h->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int grid_x = (p.nblk + kBlockThreads - 1) / kBlockThreads;
  for (int f0 = 0; f0 < n; f0 += 65535) {                    // gridDim.y is at most 65535
    const int nf = n - f0 < 65535 ? n - f0 : 65535;
    p.images = images + f0 * p.image_stride;
    p.out = out + f0 * out_stride;
    p.sizes = sizes + f0;
    p.ws = static_cast<uint8_t*>(ws) + f0 * lay.bytes;
    lspj_block_kernel<<<dim3(grid_x, nf), kBlockThreads, 0, s>>>(p);
    lspj_offsets_kernel<<<nf, kFrameThreads, 0, s>>>(p);
    lspj_pack_kernel<<<dim3(grid_x, nf), kBlockThreads, 0, s>>>(p);
    lspj_stuff_kernel<<<nf, kFrameThreads, 0, s>>>(p);
  }
  CUDA_TRY(cudaGetLastError());
  return LSPG_OK;
}

}  // extern "C"
