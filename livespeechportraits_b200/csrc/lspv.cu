// lspv.cu - the H.264 Constrained Baseline encoder of include/lspv.h.
//
// Per frame, in order on the caller's stream:
//   1. lspv_colour_kernel     RGB / grey -> BT.601 Y'CbCr 4:2:0 in the workspace.
//   2. lspv_intra_kernel      (IDR) the I_16x16 wavefront: one CTA per macroblock row, rows taken by ticket, each
//                             macroblock after its upper neighbour through a progress counter in global memory.
//      lspv_inter_kernel      (P) one CTA per macroblock: full-pel search, then prediction, transform, quantisation and
//                             reconstruction.  Reads only the previous reconstruction, so every macroblock runs at once.
//   3. lspv_bits_kernel       one thread per macroblock: P_Skip decision and the macroblock's CAVLC length.
//   4. lspv_offsets_kernel    one CTA: mb_skip_run lengths (max-scan), bit offsets (sum-scan), zeroed bit buffer.
//   5. lspv_pack_kernel       one thread per macroblock: CAVLC into the bit buffer with atomicOr.
//   6. lspv_finish_kernel     one CTA: start codes, parameter sets, NAL header, trailing bits, emulation prevention.
// then the reconstruction is copied into the caller's state.  oracle/h264_oracle.py restates every stage.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>
#include <string>

#include "../../include/lspv.h"
#include "bitstream.cuh"
#include "capi.cuh"

using bitstream::block_exclusive_scan;
using bitstream::BitWriter;
using bitstream::Max;
using bitstream::Sum;
using capi::align256;
using capi::DeviceGuard;

namespace {

struct Lspv;
constexpr auto fail = capi::fail<Lspv>;

constexpr int kThreads = 256;          // per macroblock CTA
constexpr int kFrameThreads = 1024;
constexpr int kMaxSearch = 64;
constexpr int kLevelMax = 2063;
constexpr int64_t kMaxAuBytes = int64_t(1) << 30;
constexpr int kPsBytes = 128;

// ---- tables (lspv.h; oracle/h264_oracle.py names them alike) ---------------------------------------------------------

__constant__ uint8_t kLambda[52] = {0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 4, 4,
                                    5, 5, 6, 7, 7, 8, 9, 10, 12, 13, 15, 17, 19, 21, 23, 26, 30, 33, 37, 42, 47, 53,
                                    59, 66, 74, 83};
__constant__ int kMF[6][3] = {{13107, 5243, 8066}, {11916, 4660, 7490}, {10082, 4194, 6554},
                              {9362, 3647, 5825},  {8192, 3355, 5243},  {7282, 2893, 4559}};
__constant__ int kV[6][3] = {{10, 16, 13}, {11, 18, 14}, {13, 20, 16}, {14, 23, 18}, {16, 25, 20}, {18, 29, 23}};
__constant__ uint8_t kZigzag[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};
__constant__ uint8_t kBlkX[16] = {0, 1, 0, 1, 2, 3, 2, 3, 0, 1, 0, 1, 2, 3, 2, 3};
__constant__ uint8_t kBlkY[16] = {0, 0, 1, 1, 0, 0, 1, 1, 2, 2, 3, 3, 2, 2, 3, 3};
__constant__ uint8_t kBlkOf[16] = {0, 1, 4, 5, 2, 3, 6, 7, 8, 9, 12, 13, 10, 11, 14, 15};   // [y * 4 + x]
__constant__ uint8_t kChromaQp[52] = {0,  1,  2,  3,  4,  5,  6,  7,  8,  9,  10, 11, 12, 13, 14, 15, 16, 17,
                                      18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 29, 30, 31, 32, 32, 33,
                                      34, 34, 35, 35, 36, 36, 37, 37, 37, 38, 38, 38, 39, 39, 39, 39};
__constant__ uint8_t kInterCbpCode[48] = {0,  2,  3,  7,  4,  8,  17, 13, 5,  18, 9,  14, 10, 15, 16, 11,
                                          1,  32, 33, 36, 34, 37, 44, 40, 35, 45, 38, 41, 39, 42, 43, 19,
                                          6,  24, 25, 20, 26, 21, 46, 28, 27, 47, 22, 29, 23, 30, 31, 12};
// Table 9-5 [nC class][4 TotalCoeff + TrailingOnes]
__constant__ uint8_t kCtLen[4][68] = {
    {1,  0,  0,  0,  6,  2,  0,  0,  8,  6,  3,  0,  9,  8,  7,  5,  10, 9,  8,  6,  11, 10, 9,
     7,  13, 11, 10, 8,  13, 13, 11, 9,  13, 13, 13, 10, 14, 14, 13, 11, 14, 14, 14, 13, 15, 15,
     14, 14, 15, 15, 15, 14, 16, 15, 15, 15, 16, 16, 16, 15, 16, 16, 16, 16, 16, 16, 16, 16},
    {2,  0,  0,  0,  6,  2,  0,  0,  6,  5,  3,  0,  7,  6,  6,  4,  8,  6,  6,  4,  8,  7,  7,
     5,  9,  8,  8,  6,  11, 9,  9,  6,  11, 11, 11, 7,  12, 11, 11, 9,  12, 12, 12, 11, 12, 12,
     12, 11, 13, 13, 13, 12, 13, 13, 13, 13, 13, 14, 13, 13, 14, 14, 14, 13, 14, 14, 14, 14},
    {4, 0, 0, 0, 6, 4, 0, 0, 6, 5, 4, 0, 6, 5, 5, 4, 7, 5, 5, 4, 7,  5,  5,  4,  7,  6,  6,  4, 7,  6,  6,  4,  8, 7,
     7, 5, 8, 8, 7, 6, 9, 8, 8, 7, 9, 9, 8, 8, 9, 9, 9, 8, 10, 9, 9, 9, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10},
    {6, 0, 0, 0, 6, 6, 0, 0, 6, 6, 6, 0, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6,
     6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6}};
__constant__ uint8_t kCtCode[4][68] = {
    {1,  0,  0,  0, 5,  1,  0,  0,  7, 4,  1,  0, 7, 6,  5, 3, 7,  6,  5, 3, 7, 6,  5,
     4,  15, 6,  5, 4,  11, 14, 5,  4, 8,  10, 13, 4, 15, 14, 9, 4, 11, 10, 13, 12, 15, 14,
     9,  12, 11, 10, 13, 8, 15, 1,  9, 12, 11, 14, 13, 8, 7,  10, 9, 12, 4, 6, 5,  8},
    {3, 0, 0, 0, 11, 2,  0,  0,  7,  7,  3,  0, 7,  10, 9,  5, 7, 6, 5,  4,  4,  6, 5,
     6, 7, 6, 5, 8,  15, 6,  5,  4,  11, 14, 13, 4, 15, 10, 9, 4, 11, 14, 13, 12, 8, 10,
     9, 8, 15, 14, 13, 12, 11, 10, 9,  12, 7,  11, 6,  8,  9,  8, 10, 1, 7,  6,  5,  4},
    {15, 0,  0,  0, 15, 14, 0,  0,  11, 15, 13, 0,  8,  12, 14, 12, 15, 10, 11, 11, 11, 8,  9,
     10, 9,  14, 13, 9, 8,  10, 9,  8,  15, 14, 13, 13, 11, 14, 10, 12, 15, 10, 13, 12, 11, 14,
     9,  12, 8,  10, 13, 8, 13, 7,  9,  12, 9,  12, 11, 10, 5,  8,  7,  6,  1,  4,  3,  2},
    {3,  0,  0,  0,  0,  1,  0,  0,  4,  5,  6,  0,  8,  9,  10, 11, 12, 13, 14, 15, 16, 17, 18,
     19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33, 34, 35, 36, 37, 38, 39, 40, 41,
     42, 43, 44, 45, 46, 47, 48, 49, 50, 51, 52, 53, 54, 55, 56, 57, 58, 59, 60, 61, 62, 63}};
__constant__ uint8_t kCdcLen[20] = {2, 0, 0, 0, 6, 1, 0, 0, 6, 6, 3, 0, 6, 7, 7, 6, 6, 8, 8, 7};
__constant__ uint8_t kCdcCode[20] = {1, 0, 0, 0, 7, 1, 0, 0, 4, 6, 1, 0, 3, 3, 2, 5, 2, 3, 2, 0};
// Tables 9-7, 9-8 [TotalCoeff - 1][total_zeros]
__constant__ uint8_t kTzLen[15][16] = {
    {1, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 9}, {3, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 6, 6, 6, 6},
    {4, 3, 3, 3, 4, 4, 3, 3, 4, 5, 5, 6, 5, 6},       {5, 3, 4, 4, 3, 3, 3, 4, 3, 4, 5, 5, 5},
    {4, 4, 4, 3, 3, 3, 3, 3, 4, 5, 4, 5},             {6, 5, 3, 3, 3, 3, 3, 3, 4, 3, 6},
    {6, 5, 3, 3, 3, 2, 3, 4, 3, 6},                   {6, 4, 5, 3, 2, 2, 3, 3, 6},
    {6, 6, 4, 2, 2, 3, 2, 5},                         {5, 5, 3, 2, 2, 2, 4},
    {4, 4, 3, 3, 1, 3},                               {4, 4, 2, 1, 3},
    {3, 3, 1, 2},                                     {2, 2, 1},
    {1, 1}};
__constant__ uint8_t kTzCode[15][16] = {
    {1, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 1}, {7, 6, 5, 4, 3, 5, 4, 3, 2, 3, 2, 3, 2, 1, 0},
    {5, 7, 6, 5, 4, 3, 4, 3, 2, 3, 2, 1, 1, 0},       {3, 7, 5, 4, 6, 5, 4, 3, 3, 2, 2, 1, 0},
    {5, 4, 3, 7, 6, 5, 4, 3, 2, 1, 1, 0},             {1, 1, 7, 6, 5, 4, 3, 2, 1, 1, 0},
    {1, 1, 5, 4, 3, 3, 2, 1, 1, 0},                   {1, 1, 1, 3, 3, 2, 2, 1, 0},
    {1, 0, 1, 3, 2, 1, 1, 1},                         {1, 0, 1, 3, 2, 1, 1},
    {0, 1, 1, 2, 1, 3},                               {0, 1, 1, 1, 1},
    {0, 1, 1, 1},                                     {0, 1, 1},
    {0, 1}};
__constant__ uint8_t kCtzLen[3][4] = {{1, 2, 3, 3}, {1, 2, 2, 0}, {1, 1, 0, 0}};
__constant__ uint8_t kCtzCode[3][4] = {{1, 1, 1, 0}, {1, 1, 0, 0}, {1, 0, 0, 0}};
// Table 9-10 [min(zerosLeft, 7) - 1][run_before]
__constant__ uint8_t kRbLen[7][15] = {{1, 1}, {1, 2, 2}, {2, 2, 2, 2}, {2, 2, 2, 3, 3}, {2, 2, 3, 3, 3, 3},
                                      {2, 3, 3, 3, 3, 3, 3}, {3, 3, 3, 3, 3, 3, 3, 4, 5, 6, 7, 8, 9, 10, 11}};
__constant__ uint8_t kRbCode[7][15] = {{1, 0}, {1, 1, 0}, {3, 2, 1, 0}, {3, 2, 1, 1, 0}, {3, 2, 3, 2, 1, 0},
                                       {3, 0, 1, 3, 2, 5, 4}, {7, 6, 5, 4, 3, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1}};

// Table A-1: level_idc, MaxMBPS, MaxFS, MaxDpbMbs
constexpr int64_t kLevels[19][4] = {
    {10, 1485, 99, 396},        {11, 3000, 396, 900},       {12, 6000, 396, 2376},      {13, 11880, 396, 2376},
    {20, 11880, 396, 2376},     {21, 19800, 792, 4752},     {22, 20250, 1620, 8100},    {30, 40500, 1620, 8100},
    {31, 108000, 3600, 18000},  {32, 216000, 5120, 20480},  {40, 245760, 8192, 32768},  {41, 245760, 8192, 32768},
    {42, 522240, 8704, 34816},  {50, 589824, 22080, 110400}, {51, 983040, 36864, 184320},
    {52, 2073600, 36864, 184320}, {60, 4177920, 139264, 696320}, {61, 8355840, 139264, 696320},
    {62, 16711680, 139264, 696320}};

// ---- per-macroblock record and launch parameters -----------------------------------------------------------------

struct MbRec {
  int16_t luma[16][16];      // [luma4x4BlkIdx][scan]; I_16x16 leaves [b][0] at 0 (its DC levels are `dc`)
  int16_t dc[16];            // Intra16x16DCLevel, scan order
  int16_t cdc[2][4];         // chroma DC levels, Cb then Cr, raster order of the 2x2
  int16_t cac[2][4][16];     // chroma AC levels, [comp][blk][scan], [..][0] unused
  int16_t mvx, mvy;          // quarter samples
  uint8_t tc_luma[16];       // TotalCoeff per luma4x4BlkIdx (AC only for I_16x16)
  uint8_t tc_chroma[2][4];
  uint8_t mode, cmode, cbp, skip;
};

struct Layout {               // byte offsets into the workspace
  size_t yuv, rec, mbs, bits, runs, counters, buf, bytes;
};

struct Params {
  const uint8_t* image;       // this frame's input
  uint8_t* ws;
  uint8_t* state;             // [int64 next frame][pad][Y][Cb][Cr] of the previous reconstruction
  uint8_t* out;               // this frame's slot
  int32_t* size;
  uint8_t* is_idr;
  Layout lay;
  int height, width, comps, mbw, mbh, nmb;
  int qp, search, idr;
  int64_t frame;
  int ps_len;                 // bytes of start code + SPS + start code + PPS (IDR only), emulation prevention applied
  uint8_t ps[kPsBytes];
  int sh_bits;                // slice header bits
  uint8_t sh[16];
  uint8_t nal_header;
};

constexpr size_t kStateHeader = 256;

__device__ __forceinline__ uint8_t* yuv_plane(const Params& p, int c) {
  const size_t hw = static_cast<size_t>(p.height) * p.width;
  return p.ws + p.lay.yuv + (c == 0 ? 0 : c == 1 ? hw : hw + hw / 4);
}
__device__ __forceinline__ uint8_t* rec_plane(const Params& p, int c) {
  const size_t hw = static_cast<size_t>(p.height) * p.width;
  return p.ws + p.lay.rec + (c == 0 ? 0 : c == 1 ? hw : hw + hw / 4);
}
__device__ __forceinline__ const uint8_t* ref_plane(const Params& p, int c) {
  const size_t hw = static_cast<size_t>(p.height) * p.width;
  return p.state + kStateHeader + (c == 0 ? 0 : c == 1 ? hw : hw + hw / 4);
}
__device__ __forceinline__ MbRec* mb_recs(const Params& p) { return reinterpret_cast<MbRec*>(p.ws + p.lay.mbs); }
__device__ __forceinline__ uint32_t* mb_bits(const Params& p) { return reinterpret_cast<uint32_t*>(p.ws + p.lay.bits); }
__device__ __forceinline__ uint32_t* mb_runs(const Params& p) { return reinterpret_cast<uint32_t*>(p.ws + p.lay.runs); }
__device__ __forceinline__ int* counters(const Params& p) { return reinterpret_cast<int*>(p.ws + p.lay.counters); }
__device__ __forceinline__ uint32_t* bit_buf(const Params& p) { return reinterpret_cast<uint32_t*>(p.ws + p.lay.buf); }

__device__ __forceinline__ int clip255(int v) { return v < 0 ? 0 : v > 255 ? 255 : v; }
__device__ __forceinline__ int cls(int i) { return ((i >> 2) & 1) == 0 && (i & 1) == 0 ? 0 : ((i >> 2) & 1) && (i & 1) ? 1 : 2; }

// ---- 1. colour ------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kThreads) lspv_colour_kernel(const Params p) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  const int wc = p.width / 2, hc = p.height / 2;
  if (i >= wc * hc) return;
  const int cx = i % wc, cy = i / wc;
  int sb = 0, sr = 0;
  uint8_t* y = yuv_plane(p, 0);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int px = 2 * cx + (k & 1), py = 2 * cy + (k >> 1);
    const size_t at = static_cast<size_t>(py) * p.width + px;
    int r, g, b;
    if (p.comps == 3) {
      r = p.image[3 * at], g = p.image[3 * at + 1], b = p.image[3 * at + 2];
    } else {
      r = g = b = p.image[at];
    }
    y[at] = static_cast<uint8_t>(((66 * r + 129 * g + 25 * b + 128) >> 8) + 16);
    sb += ((-38 * r - 74 * g + 112 * b + 128) >> 8) + 128;
    sr += ((112 * r - 94 * g - 18 * b + 128) >> 8) + 128;
  }
  yuv_plane(p, 1)[i] = static_cast<uint8_t>((sb + 2) >> 2);
  yuv_plane(p, 2)[i] = static_cast<uint8_t>((sr + 2) >> 2);
}

// ---- shared macroblock coding: transform, quantisation, scaling, reconstruction (8.5) ------------------------------

struct MbShared {
  int16_t pred[384];          // luma 16x16, Cb 8x8, Cr 8x8
  int32_t coef[24][16];       // forward-transformed blocks: luma by blkIdx, then Cb 0..3, Cr 0..3 (raster)
  int32_t dc[3][16];          // scaled DC values: dcY by blkIdx, dcC by raster block
  int32_t sums[8];
  uint32_t key;
  int mode, cmode;
};

__device__ __forceinline__ void forward4(const int* r, int32_t* w) {
  int t[16];
#pragma unroll
  for (int i = 0; i < 4; ++i) {                                  // rows: Cf x
    const int a = r[4 * i], b = r[4 * i + 1], c = r[4 * i + 2], d = r[4 * i + 3];
    const int s0 = a + d, s1 = b + c, d0 = a - d, d1 = b - c;
    t[4 * i] = s0 + s1, t[4 * i + 1] = 2 * d0 + d1, t[4 * i + 2] = s0 - s1, t[4 * i + 3] = d0 - 2 * d1;
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {                                  // columns
    const int a = t[j], b = t[4 + j], c = t[8 + j], d = t[12 + j];
    const int s0 = a + d, s1 = b + c, d0 = a - d, d1 = b - c;
    w[j] = s0 + s1, w[4 + j] = 2 * d0 + d1, w[8 + j] = s0 - s1, w[12 + j] = d0 - 2 * d1;
  }
}

__device__ __forceinline__ int quant(int w, int mf, int shift, int f) {
  int z = static_cast<int>((static_cast<int64_t>(w < 0 ? -w : w) * mf + f) >> shift);
  z = z > kLevelMax ? kLevelMax : z;
  return w < 0 ? -z : z;
}

__device__ __forceinline__ void inverse4(int* d) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int* r = d + 4 * i;
    const int e0 = r[0] + r[2], e1 = r[0] - r[2], e2 = (r[1] >> 1) - r[3], e3 = r[1] + (r[3] >> 1);
    r[0] = e0 + e3, r[1] = e1 + e2, r[2] = e1 - e2, r[3] = e0 - e3;
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int g0 = d[j], g1 = d[4 + j], g2 = d[8 + j], g3 = d[12 + j];
    const int e0 = g0 + g2, e1 = g0 - g2, e2 = (g1 >> 1) - g3, e3 = g1 + (g3 >> 1);
    d[j] = (e0 + e3 + 32) >> 6, d[4 + j] = (e1 + e2 + 32) >> 6, d[8 + j] = (e1 - e2 + 32) >> 6,
    d[12 + j] = (e0 - e3 + 32) >> 6;
  }
}

// Codes macroblock (mx, my) from the source planes and s.pred into rec (levels, TotalCoeff, cbp) and the
// reconstruction planes.  All kThreads threads call it.
__device__ void code_mb(const Params& p, MbShared& s, MbRec* rec, int mx, int my, bool intra) {
  const int t = threadIdx.x;
  const int qp = p.qp, qpc = kChromaQp[p.qp];
  const int f4 = (1 << (15 + qp / 6)) / (intra ? 3 : 6), f4c = (1 << (15 + qpc / 6)) / (intra ? 3 : 6);
  if (t < 24) {                                                   // residual + forward transform of one 4x4 block
    int r[16];
    if (t < 16) {
      const int bx = kBlkX[t], by = kBlkY[t];
      const uint8_t* src = yuv_plane(p, 0) + static_cast<size_t>(16 * my + 4 * by) * p.width + 16 * mx + 4 * bx;
#pragma unroll
      for (int k = 0; k < 16; ++k) r[k] = src[(k >> 2) * p.width + (k & 3)] - s.pred[(4 * by + (k >> 2)) * 16 + 4 * bx + (k & 3)];
    } else {
      const int c = (t - 16) >> 2, b = (t - 16) & 3, bx = b & 1, by = b >> 1, wc = p.width / 2;
      const uint8_t* src = yuv_plane(p, 1 + c) + static_cast<size_t>(8 * my + 4 * by) * wc + 8 * mx + 4 * bx;
      const int16_t* pr = s.pred + 256 + 64 * c;
#pragma unroll
      for (int k = 0; k < 16; ++k) r[k] = src[(k >> 2) * wc + (k & 3)] - pr[(4 * by + (k >> 2)) * 8 + 4 * bx + (k & 3)];
    }
    forward4(r, s.coef[t]);
  }
  __syncthreads();
  if (t < 24) {                                                   // AC (and inter luma DC) levels, TotalCoeff
    const bool chroma = t >= 16;
    const int q = chroma ? qpc : qp, mfi = q % 6, shift = 15 + q / 6, f = chroma ? f4c : f4;
    const bool skip_dc = chroma || intra;
    int16_t* lev = chroma ? rec->cac[(t - 16) >> 2][(t - 16) & 3] : rec->luma[t];
    int nz = 0;
    for (int k = 0; k < 16; ++k) {
      const int i = kZigzag[k];
      const int z = (k == 0 && skip_dc) ? 0 : quant(s.coef[t][i], kMF[mfi][cls(i)], shift, f);
      lev[k] = static_cast<int16_t>(z);
      nz += z != 0;
    }
    if (chroma) rec->tc_chroma[(t - 16) >> 2][(t - 16) & 3] = static_cast<uint8_t>(nz);
    else rec->tc_luma[t] = static_cast<uint8_t>(nz);
  } else if (t == 32 && intra) {                                 // luma DC: Hadamard, halved, quantised, scaled (8.5.10)
    int d[16], h[16];
    for (int k = 0; k < 16; ++k) d[k] = s.coef[kBlkOf[k]][0];     // [block y][block x]
    for (int i = 0; i < 4; ++i) {
      const int a = d[4 * i], b = d[4 * i + 1], c = d[4 * i + 2], e = d[4 * i + 3];
      h[4 * i] = a + b + c + e, h[4 * i + 1] = a + b - c - e, h[4 * i + 2] = a - b - c + e, h[4 * i + 3] = a - b + c - e;
    }
    for (int j = 0; j < 4; ++j) {
      const int a = h[j], b = h[4 + j], c = h[8 + j], e = h[12 + j];
      d[j] = (a + b + c + e) >> 1, d[4 + j] = (a + b - c - e) >> 1, d[8 + j] = (a - b - c + e) >> 1,
      d[12 + j] = (a - b + c - e) >> 1;
    }
    const int shift = 16 + qp / 6;
    for (int k = 0; k < 16; ++k) d[k] = quant(d[k], kMF[qp % 6][0], shift, 2 * f4);
    for (int k = 0; k < 16; ++k) rec->dc[k] = static_cast<int16_t>(d[kZigzag[k]]);
    for (int i = 0; i < 4; ++i) {
      const int a = d[4 * i], b = d[4 * i + 1], c = d[4 * i + 2], e = d[4 * i + 3];
      h[4 * i] = a + b + c + e, h[4 * i + 1] = a + b - c - e, h[4 * i + 2] = a - b - c + e, h[4 * i + 3] = a - b + c - e;
    }
    const int ls = 16 * kV[qp % 6][0];
    for (int j = 0; j < 4; ++j) {
      const int a = h[j], b = h[4 + j], c = h[8 + j], e = h[12 + j];
      const int f[4] = {a + b + c + e, a + b - c - e, a - b - c + e, a - b + c - e};
      for (int i = 0; i < 4; ++i) {
        const int v = qp >= 36 ? (f[i] * ls) << (qp / 6 - 6) : (f[i] * ls + (1 << (5 - qp / 6))) >> (6 - qp / 6);
        s.dc[0][kBlkOf[4 * i + j]] = v;
      }
    }
  } else if (t == 64 || t == 65) {                               // chroma DC: 2x2 transform, quantised, scaled (8.5.11)
    const int c = t - 64;
    const int* w0 = s.coef[16 + 4 * c];
    const int a = w0[0], b = s.coef[17 + 4 * c][0], cc = s.coef[18 + 4 * c][0], d = s.coef[19 + 4 * c][0];
    int z[4] = {a + b + cc + d, a - b + cc - d, a + b - cc - d, a - b - cc + d};
    const int shift = 16 + qpc / 6;
    for (int k = 0; k < 4; ++k) {
      z[k] = quant(z[k], kMF[qpc % 6][0], shift, 2 * f4c);
      rec->cdc[c][k] = static_cast<int16_t>(z[k]);
    }
    const int f[4] = {z[0] + z[1] + z[2] + z[3], z[0] - z[1] + z[2] - z[3], z[0] + z[1] - z[2] - z[3],
                      z[0] - z[1] - z[2] + z[3]};
    const int ls = 16 * kV[qpc % 6][0];
    for (int k = 0; k < 4; ++k) s.dc[1 + c][k] = ((f[k] * ls) << (qpc / 6)) >> 5;
  }
  __syncthreads();
  if (t < 24) {                                                   // scaling, inverse transform, reconstruction
    const bool chroma = t >= 16;
    const int q = chroma ? qpc : qp;
    const int16_t* lev = chroma ? rec->cac[(t - 16) >> 2][(t - 16) & 3] : rec->luma[t];
    int d[16];
    for (int k = 0; k < 16; ++k) {
      const int i = kZigzag[k];
      d[i] = (lev[k] * kV[q % 6][cls(i)]) << (q / 6);
    }
    if (chroma) d[0] = s.dc[1 + ((t - 16) >> 2)][(t - 16) & 3];
    else if (intra) d[0] = s.dc[0][t];
    inverse4(d);
    if (t < 16) {
      const int bx = kBlkX[t], by = kBlkY[t];
      uint8_t* dst = rec_plane(p, 0) + static_cast<size_t>(16 * my + 4 * by) * p.width + 16 * mx + 4 * bx;
      for (int k = 0; k < 16; ++k)
        dst[(k >> 2) * p.width + (k & 3)] =
            static_cast<uint8_t>(clip255(s.pred[(4 * by + (k >> 2)) * 16 + 4 * bx + (k & 3)] + d[k]));
    } else {
      const int c = (t - 16) >> 2, b = (t - 16) & 3, bx = b & 1, by = b >> 1, wc = p.width / 2;
      uint8_t* dst = rec_plane(p, 1 + c) + static_cast<size_t>(8 * my + 4 * by) * wc + 8 * mx + 4 * bx;
      const int16_t* pr = s.pred + 256 + 64 * c;
      for (int k = 0; k < 16; ++k)
        dst[(k >> 2) * wc + (k & 3)] = static_cast<uint8_t>(clip255(pr[(4 * by + (k >> 2)) * 8 + 4 * bx + (k & 3)] + d[k]));
    }
  }
  __syncthreads();
  if (t == 0) {
    int cbpl = 0, ac = 0, dcnz = 0;
    for (int b = 0; b < 16; ++b)
      if (rec->tc_luma[b]) cbpl |= intra ? 15 : 1 << (b >> 2);
    for (int k = 0; k < 8; ++k) ac |= rec->tc_chroma[k >> 2][k & 3];
    for (int k = 0; k < 8; ++k) dcnz |= rec->cdc[k >> 2][k & 3];
    rec->cbp = static_cast<uint8_t>(cbpl | (ac ? 2 : dcnz ? 1 : 0) << 4);
    rec->skip = 0;
  }
}

// ---- 2a. I frames: the intra wavefront (8.3.3, 8.3.4) ----------------------------------------------------------------

__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(kThreads) lspv_intra_kernel(const Params p) {
  __shared__ MbShared s;
  __shared__ int nb[3][34];          // [plane][0]: top-left, [1..16 / 8]: top, [17..32 / 9..16]: left
  __shared__ int prm[3][4];          // plane a, b, c per plane; DC values
  __shared__ int row;
  const int t = threadIdx.x;
  int* ctr = counters(p);
  if (t == 0) row = atomicAdd(ctr, 1);                           // rows start in order, so no CTA waits on one unstarted
  __syncthreads();
  const int my = row;
  volatile int* progress = ctr + 1;
  for (int mx = 0; mx < p.mbw; ++mx) {
    if (t == 0 && my > 0) {
      while (progress[my - 1] <= mx) {
      }
      __threadfence();
    }
    __syncthreads();
    const bool top = my > 0, left = mx > 0;
    if (t < 33) {                                                 // luma neighbours
      const uint8_t* y = rec_plane(p, 0);
      const int x0 = 16 * mx, y0 = 16 * my;
      int v = 0;
      if (t == 0 && top && left) v = __ldcg(y + static_cast<size_t>(y0 - 1) * p.width + x0 - 1);
      else if (t >= 1 && t <= 16 && top) v = __ldcg(y + static_cast<size_t>(y0 - 1) * p.width + x0 + t - 1);
      else if (t >= 17 && left) v = __ldcg(y + static_cast<size_t>(y0 + t - 17) * p.width + x0 - 1);
      nb[0][t] = v;
    } else if (t >= 64 && t < 64 + 34) {                          // chroma neighbours
      const int c = (t - 64) / 17, k = (t - 64) % 17, wc = p.width / 2;
      const uint8_t* pl = rec_plane(p, 1 + c);
      const int x0 = 8 * mx, y0 = 8 * my;
      int v = 0;
      if (k == 0 && top && left) v = __ldcg(pl + static_cast<size_t>(y0 - 1) * wc + x0 - 1);
      else if (k >= 1 && k <= 8 && top) v = __ldcg(pl + static_cast<size_t>(y0 - 1) * wc + x0 + k - 1);
      else if (k >= 9 && left) v = __ldcg(pl + static_cast<size_t>(y0 + k - 9) * wc + x0 - 1);
      nb[1 + c][k] = v;
    }
    if (t < 8) s.sums[t] = 0;
    __syncthreads();
    if (t < 3) {                                                  // plane parameters and (luma) DC
      const int* q = nb[t];
      if (t == 0) {
        int h = 0, v = 0;
        for (int i = 0; i < 8; ++i) h += (i + 1) * (q[9 + i] - q[7 - i]), v += (i + 1) * (q[17 + 8 + i] - (i == 7 ? q[0] : q[17 + 6 - i]));
        prm[0][0] = 16 * (q[32] + q[16]), prm[0][1] = (5 * h + 32) >> 6, prm[0][2] = (5 * v + 32) >> 6;
        int st = 0, sl = 0;
        for (int i = 0; i < 16; ++i) st += q[1 + i], sl += q[17 + i];
        prm[0][3] = top && left ? (st + sl + 16) >> 5 : left ? (sl + 8) >> 4 : top ? (st + 8) >> 4 : 128;
      } else {
        int h = 0, v = 0;
        for (int i = 0; i < 4; ++i) h += (i + 1) * (q[5 + i] - q[3 - i]), v += (i + 1) * (q[9 + 4 + i] - (i == 3 ? q[0] : q[9 + 2 - i]));
        prm[t][0] = 16 * (q[16] + q[8]), prm[t][1] = (34 * h + 32) >> 6, prm[t][2] = (34 * v + 32) >> 6;
      }
    }
    __syncthreads();
    // candidate predictions and their SADs: luma by 256 threads, chroma (both components) by the first 128
    auto luma_pred = [&](int mode, int x, int y) -> int {
      if (mode == 0) return nb[0][1 + x];
      if (mode == 1) return nb[0][17 + y];
      if (mode == 2) return prm[0][3];
      return clip255((prm[0][0] + prm[0][1] * (x - 7) + prm[0][2] * (y - 7) + 16) >> 5);
    };
    auto chroma_pred = [&](int c, int mode, int x, int y) -> int {
      const int* q = nb[1 + c];
      if (mode == 1) return q[9 + y];
      if (mode == 2) return q[1 + x];
      if (mode == 3) return clip255((prm[1 + c][0] + prm[1 + c][1] * (x - 3) + prm[1 + c][2] * (y - 3) + 16) >> 5);
      const int bx = x >> 2, by = y >> 2;
      int st = 0, sl = 0;
      for (int i = 0; i < 4; ++i) st += q[1 + 4 * bx + i], sl += q[9 + 4 * by + i];
      if (bx == by) return top && left ? (st + sl + 4) >> 3 : left ? (sl + 2) >> 2 : top ? (st + 2) >> 2 : 128;
      if (by == 0) return top ? (st + 2) >> 2 : left ? (sl + 2) >> 2 : 128;
      return left ? (sl + 2) >> 2 : top ? (st + 2) >> 2 : 128;
    };
    {
      const int x = t & 15, y = t >> 4;
      const int src = yuv_plane(p, 0)[static_cast<size_t>(16 * my + y) * p.width + 16 * mx + x];
      for (int m = 0; m < 4; ++m) {
        const int v = warp_sum(abs(src - luma_pred(m, x, y)));
        if ((t & 31) == 0) atomicAdd(&s.sums[m], v);
      }
      if (t < 128) {
        const int c = t >> 6, cx = t & 7, cy = (t >> 3) & 7, wc = p.width / 2;
        const int cs = yuv_plane(p, 1 + c)[static_cast<size_t>(8 * my + cy) * wc + 8 * mx + cx];
        for (int m = 0; m < 4; ++m) {
          const int v = warp_sum(abs(cs - chroma_pred(c, m, cx, cy)));
          if ((t & 31) == 0) atomicAdd(&s.sums[4 + m], v);
        }
      }
    }
    __syncthreads();
    if (t == 0) {
      const bool ok[4] = {top, left, true, top && left};          // V, H, DC, Plane
      const bool cok[4] = {true, left, top, top && left};         // DC, H, V, Plane
      int best = 2, cbest = 0;
      for (int m = 0; m < 4; ++m)
        if (ok[m] && (s.sums[m] < s.sums[best] || (s.sums[m] == s.sums[best] && m < best))) best = m;
      for (int m = 0; m < 4; ++m)
        if (cok[m] && (s.sums[4 + m] < s.sums[4 + cbest] || (s.sums[4 + m] == s.sums[4 + cbest] && m < cbest))) cbest = m;
      s.mode = best, s.cmode = cbest;
    }
    __syncthreads();
    s.pred[t] = static_cast<int16_t>(luma_pred(s.mode, t & 15, t >> 4));
    if (t < 128) s.pred[256 + t] = static_cast<int16_t>(chroma_pred(t >> 6, s.cmode, t & 7, (t >> 3) & 7));
    __syncthreads();
    MbRec* rec = mb_recs(p) + my * p.mbw + mx;
    code_mb(p, s, rec, mx, my, true);
    __threadfence();                                              // this macroblock's reconstruction, then its flag
    __syncthreads();
    if (t == 0) {
      rec->mode = static_cast<uint8_t>(s.mode), rec->cmode = static_cast<uint8_t>(s.cmode);
      rec->mvx = rec->mvy = 0;
      progress[my] = mx + 1;
    }
  }
}

// ---- 2b. P frames: motion search and inter coding (8.4) --------------------------------------------------------------

__device__ __forceinline__ int se_bits(int v) {
  const unsigned k = v > 0 ? 2u * v - 1 : 2u * static_cast<unsigned>(-v);
  return 2 * (32 - __clz(k + 1)) - 1;
}

__global__ void __launch_bounds__(kThreads) lspv_inter_kernel(const Params p) {
  __shared__ MbShared s;
  extern __shared__ uint32_t win[];                              // reference window, (16 + 2 search) rows, pitch in words
  __shared__ uint32_t cur[64];
  const int t = threadIdx.x, mx = blockIdx.x, my = blockIdx.y;
  const int S = p.search, span = 16 + 2 * S, pitch = (span + 3) / 4 + 1;
  const int x0 = 16 * mx, y0 = 16 * my;
  const uint8_t* ref = ref_plane(p, 0);
  uint8_t* wb = reinterpret_cast<uint8_t*>(win);
  for (int i = t; i < span * pitch * 4; i += kThreads) {
    const int r = i / (pitch * 4), c = i % (pitch * 4);
    const int yy = min(max(y0 - S + r, 0), p.height - 1), xx = min(max(x0 - S + c, 0), p.width - 1);
    wb[i] = ref[static_cast<size_t>(yy) * p.width + xx];
  }
  if (t < 64) {
    const uint8_t* src = yuv_plane(p, 0) + static_cast<size_t>(y0 + (t >> 2)) * p.width + x0 + 4 * (t & 3);
    cur[t] = src[0] | src[1] << 8 | src[2] << 16 | static_cast<uint32_t>(src[3]) << 24;
  }
  if (t == 0) s.key = 0xffffffffu;
  __syncthreads();
  const int lo_x = max(-S, -x0), hi_x = min(S, p.width - 16 - x0);
  const int lo_y = max(-S, -y0), hi_y = min(S, p.height - 16 - y0);
  const int side = 2 * S + 1, lam = kLambda[p.qp];
  uint32_t best = 0xffffffffu;
  for (int idx = t; idx < side * side; idx += kThreads) {
    const int dy = idx / side - S, dx = idx % side - S;
    if (dx < lo_x || dx > hi_x || dy < lo_y || dy > hi_y) continue;
    uint32_t sad = 0;
    const int bx = dx + S, sh = 8 * (bx & 3);
    for (int r = 0; r < 16; ++r) {
      const uint32_t* w = win + (r + dy + S) * pitch + (bx >> 2);
      const uint32_t w0 = w[0], w1 = w[1], w2 = w[2], w3 = w[3], w4 = w[4];
      sad += __vsadu4(cur[4 * r], __funnelshift_r(w0, w1, sh));
      sad += __vsadu4(cur[4 * r + 1], __funnelshift_r(w1, w2, sh));
      sad += __vsadu4(cur[4 * r + 2], __funnelshift_r(w2, w3, sh));
      sad += __vsadu4(cur[4 * r + 3], __funnelshift_r(w3, w4, sh));
    }
    const uint32_t cost = sad + lam * (se_bits(4 * dx) + se_bits(4 * dy));
    const uint32_t key = cost << 15 | static_cast<uint32_t>(idx);
    best = min(best, key);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
  if ((t & 31) == 0) atomicMin(&s.key, best);
  __syncthreads();
  const int idx = s.key & 0x7fff;
  const int dy = idx / side - S, dx = idx % side - S;
  {                                                               // luma prediction: full-pel, inside the frame
    const int x = t & 15, y = t >> 4;
    s.pred[t] = ref[static_cast<size_t>(y0 + dy + y) * p.width + x0 + dx + x];
  }
  if (t < 128) {                                                  // chroma: eighth-sample bilinear with clamping
    const int c = t >> 6, cx = t & 7, cy = (t >> 3) & 7, wc = p.width / 2, hc = p.height / 2;
    const uint8_t* rp = ref_plane(p, 1 + c);
    const int fx = (4 * dx) & 7, fy = (4 * dy) & 7;
    const int xi = 8 * mx + ((4 * dx) >> 3) + cx, yi = 8 * my + ((4 * dy) >> 3) + cy;
    const int xa = min(max(xi, 0), wc - 1), xb = min(max(xi + 1, 0), wc - 1);
    const int ya = min(max(yi, 0), hc - 1), yb = min(max(yi + 1, 0), hc - 1);
    const int A = rp[static_cast<size_t>(ya) * wc + xa], B = rp[static_cast<size_t>(ya) * wc + xb];
    const int C = rp[static_cast<size_t>(yb) * wc + xa], D = rp[static_cast<size_t>(yb) * wc + xb];
    s.pred[256 + t] = static_cast<int16_t>(((8 - fx) * (8 - fy) * A + fx * (8 - fy) * B + (8 - fx) * fy * C + fx * fy * D + 32) >> 6);
  }
  __syncthreads();
  MbRec* rec = mb_recs(p) + my * p.mbw + mx;
  code_mb(p, s, rec, mx, my, false);
  if (t == 0) {
    rec->mvx = static_cast<int16_t>(4 * dx), rec->mvy = static_cast<int16_t>(4 * dy);
    rec->mode = rec->cmode = 0;
  }
}

// ---- 3-5. CAVLC ---------------------------------------------------------------------------------------------------

struct Counter {
  uint32_t n = 0;
  __device__ __forceinline__ void put(uint32_t, int size) { n += size; }
};

template <class W>
__device__ __forceinline__ void put_ue(W& w, uint32_t v) {
  const int k = 32 - __clz(v + 1);
  w.put(0, k - 1);
  w.put(v + 1, k);
}
template <class W>
__device__ __forceinline__ void put_se(W& w, int v) {
  put_ue(w, v > 0 ? 2u * v - 1 : 2u * static_cast<uint32_t>(-v));
}

// residual_block_cavlc (9.2) of n levels in scan order with context nc (-1: chroma DC)
template <class W>
__device__ void residual_block(W& w, const int16_t* coef, int n, int nc) {
  int tc = 0, last = -1;
  for (int i = 0; i < n; ++i)
    if (coef[i]) ++tc, last = i;
  int t1 = 0;
  for (int i = last; i >= 0 && t1 < 3; --i) {
    if (!coef[i]) continue;
    if (coef[i] != 1 && coef[i] != -1) break;
    ++t1;
  }
  if (nc == -1) {
    w.put(kCdcCode[4 * tc + t1], kCdcLen[4 * tc + t1]);
  } else {
    const int k = nc < 2 ? 0 : nc < 4 ? 1 : nc < 8 ? 2 : 3;
    w.put(kCtCode[k][4 * tc + t1], kCtLen[k][4 * tc + t1]);
  }
  if (!tc) return;
  int sl = tc > 10 && t1 < 3 ? 1 : 0, k = 0;
  for (int i = last; i >= 0; --i) {
    const int lv = coef[i];
    if (!lv) continue;
    if (k < t1) {
      w.put(lv < 0, 1);
    } else {
      int code = lv > 0 ? 2 * lv - 2 : -2 * lv - 1;
      if (k == t1 && t1 < 3) code -= 2;
      int prefix, suffix, size;
      if (sl == 0) {
        if (code < 14) prefix = code, suffix = 0, size = 0;
        else if (code < 30) prefix = 14, suffix = code - 14, size = 4;
        else prefix = 15, suffix = code - 30, size = 12;
      } else if (code < (15 << sl)) {
        prefix = code >> sl, suffix = code & ((1 << sl) - 1), size = sl;
      } else {
        prefix = 15, suffix = code - (15 << sl), size = 12;
      }
      w.put(1, prefix + 1);
      w.put(suffix, size);
      if (sl == 0) sl = 1;
      if ((lv < 0 ? -lv : lv) > (3 << (sl - 1)) && sl < 6) ++sl;
    }
    ++k;
  }
  const int tz = last + 1 - tc;
  if (tc < n) {
    if (n == 4) w.put(kCtzCode[tc - 1][tz], kCtzLen[tc - 1][tz]);
    else w.put(kTzCode[tc - 1][tz], kTzLen[tc - 1][tz]);
  }
  int left = tz, at = last;
  for (int c = tc - 1; c > 0 && left > 0; --c) {
    int prev = at - 1;
    while (!coef[prev]) --prev;
    const int run = at - prev - 1, r = (left < 7 ? left : 7) - 1;
    w.put(kRbCode[r][run], kRbLen[r][run]);
    left -= run;
    at = prev;
  }
}

__device__ __forceinline__ int nc_of(int a, int b) {              // -1: unavailable
  if (a >= 0 && b >= 0) return (a + b + 1) >> 1;
  return a >= 0 ? a : b >= 0 ? b : 0;
}

// TotalCoeff of the luma 4x4 block at (X, Y) in 4x4 units of the frame, -1 outside it
__device__ __forceinline__ int tc_luma_at(const Params& p, const MbRec* m, int X, int Y) {
  if (X < 0 || Y < 0) return -1;
  return m[(Y >> 2) * p.mbw + (X >> 2)].tc_luma[kBlkOf[(Y & 3) * 4 + (X & 3)]];
}
__device__ __forceinline__ int tc_chroma_at(const Params& p, const MbRec* m, int c, int X, int Y) {
  if (X < 0 || Y < 0) return -1;
  return m[(Y >> 1) * p.mbw + (X >> 1)].tc_chroma[c][(Y & 1) * 2 + (X & 1)];
}

__device__ __forceinline__ int median3(int a, int b, int c) { return max(min(a, b), min(max(a, b), c)); }

// mvp (8.4.1.3) and the P_Skip vector (8.4.1.1) of macroblock (mx, my), in quarter samples
__device__ void mv_pred(const Params& p, const MbRec* m, int mx, int my, int* mvp, int* skip) {
  auto avail = [&](int x, int y) { return x >= 0 && y >= 0 && x < p.mbw && y < p.mbh; };
  const bool ha = avail(mx - 1, my), hb = avail(mx, my - 1);
  int cx = mx + 1, cy = my - 1;
  bool hc = avail(cx, cy);
  if (!hc) cx = mx - 1, hc = avail(cx, cy);
  int a[2] = {0, 0}, b[2] = {0, 0}, c[2] = {0, 0};
  if (ha) a[0] = m[my * p.mbw + mx - 1].mvx, a[1] = m[my * p.mbw + mx - 1].mvy;
  if (hb) b[0] = m[(my - 1) * p.mbw + mx].mvx, b[1] = m[(my - 1) * p.mbw + mx].mvy;
  if (hc) c[0] = m[cy * p.mbw + cx].mvx, c[1] = m[cy * p.mbw + cx].mvy;
  bool eb = hb, ec = hc;
  if (!hb && !hc && ha) {
    b[0] = c[0] = a[0], b[1] = c[1] = a[1];
    eb = ec = true;
  }
  const int navail = ha + eb + ec;
  if (navail == 1) {
    const int* only = ha ? a : eb ? b : c;
    mvp[0] = only[0], mvp[1] = only[1];
  } else {
    mvp[0] = median3(a[0], b[0], c[0]), mvp[1] = median3(a[1], b[1], c[1]);
  }
  int ra[2] = {0, 0}, rb[2] = {0, 0};
  if (ha) ra[0] = m[my * p.mbw + mx - 1].mvx, ra[1] = m[my * p.mbw + mx - 1].mvy;
  if (hb) rb[0] = m[(my - 1) * p.mbw + mx].mvx, rb[1] = m[(my - 1) * p.mbw + mx].mvy;
  if (!ha || !hb || (ra[0] == 0 && ra[1] == 0) || (rb[0] == 0 && rb[1] == 0)) skip[0] = skip[1] = 0;
  else skip[0] = mvp[0], skip[1] = mvp[1];
}

// macroblock_layer() of macroblock i without its mb_skip_run; nothing for a P_Skip macroblock
template <class W>
__device__ void write_mb(W& w, const Params& p, const MbRec* m, int i) {
  const MbRec& r = m[i];
  const int mx = i % p.mbw, my = i / p.mbw;
  const int cbpl = r.cbp & 15, cbpc = r.cbp >> 4;
  if (p.idr) {
    put_ue(w, 1 + r.mode + 4 * cbpc + (cbpl ? 12 : 0));
    put_ue(w, r.cmode);
    put_se(w, 0);
    residual_block(w, r.dc, 16, nc_of(tc_luma_at(p, m, 4 * mx - 1, 4 * my), tc_luma_at(p, m, 4 * mx, 4 * my - 1)));
    if (cbpl)
      for (int b = 0; b < 16; ++b) {
        const int X = 4 * mx + kBlkX[b], Y = 4 * my + kBlkY[b];
        residual_block(w, r.luma[b] + 1, 15, nc_of(tc_luma_at(p, m, X - 1, Y), tc_luma_at(p, m, X, Y - 1)));
      }
  } else {
    if (r.skip) return;
    int mvp[2], skip[2];
    mv_pred(p, m, mx, my, mvp, skip);
    put_ue(w, 0);
    put_se(w, r.mvx - mvp[0]);
    put_se(w, r.mvy - mvp[1]);
    put_ue(w, kInterCbpCode[r.cbp]);
    if (!r.cbp) return;
    put_se(w, 0);
    for (int b = 0; b < 16; ++b) {
      if (!(cbpl >> (b >> 2) & 1)) continue;
      const int X = 4 * mx + kBlkX[b], Y = 4 * my + kBlkY[b];
      residual_block(w, r.luma[b], 16, nc_of(tc_luma_at(p, m, X - 1, Y), tc_luma_at(p, m, X, Y - 1)));
    }
  }
  if (cbpc)
    for (int c = 0; c < 2; ++c) residual_block(w, r.cdc[c], 4, -1);
  if (cbpc == 2)
    for (int c = 0; c < 2; ++c)
      for (int b = 0; b < 4; ++b) {
        const int X = 2 * mx + (b & 1), Y = 2 * my + (b >> 1);
        residual_block(w, r.cac[c][b] + 1, 15,
                       nc_of(tc_chroma_at(p, m, c, X - 1, Y), tc_chroma_at(p, m, c, X, Y - 1)));
      }
}

__global__ void __launch_bounds__(128) lspv_bits_kernel(const Params p) {
  const int i = blockIdx.x * 128 + threadIdx.x;
  if (i >= p.nmb) return;
  MbRec* m = mb_recs(p);
  if (!p.idr) {
    int mvp[2], skip[2];
    mv_pred(p, m, i % p.mbw, i / p.mbw, mvp, skip);
    m[i].skip = m[i].cbp == 0 && m[i].mvx == skip[0] && m[i].mvy == skip[1];
  }
  Counter c;
  write_mb(c, p, m, i);
  mb_bits(p)[i] = c.n;
}

__device__ __forceinline__ uint32_t ue_bits(uint32_t v) { return 2 * (32 - __clz(v + 1)) - 1; }

// mb_skip_run before each coded macroblock (and after the last one when the slice ends in skips), bit offsets, zeroed
// buffer.  runs[i] is the mb_skip_run macroblock i writes first (P slices), ~0u for none.
__global__ void __launch_bounds__(kFrameThreads) lspv_offsets_kernel(const Params p) {
  const MbRec* m = mb_recs(p);
  uint32_t* bits = mb_bits(p);
  uint32_t* runs = mb_runs(p);
  const bitstream::Chunk c(p.nmb);
  int last = -1;
  if (!p.idr)
    for (int i = c.i0; i < c.i1; ++i)
      if (!m[i].skip) last = i;
  int total;
  int prev = block_exclusive_scan<Max>(last, &total);
  const uint32_t end = bitstream::counts_to_offsets(bits, p.nmb, p.sh_bits, [&](int i) -> int {
    uint32_t run = ~0u;
    if (!p.idr) {
      if (!m[i].skip) run = i - prev - 1, prev = i;
      else if (i == p.nmb - 1) run = i - prev;
    }
    runs[i] = run;
    return run != ~0u ? ue_bits(run) : 0;
  });
  uint32_t* buf = bit_buf(p);
  const uint32_t words = (end + 8 + 31) / 32 + 4;
  for (uint32_t i = threadIdx.x; i < words; i += kFrameThreads) buf[i] = 0;
}

__global__ void __launch_bounds__(128) lspv_pack_kernel(const Params p) {
  const int i = blockIdx.x * 128 + threadIdx.x;
  if (i >= p.nmb) return;
  const MbRec* m = mb_recs(p);
  uint32_t* buf = bit_buf(p);
  if (i == 0) {                                                   // the slice header
    BitWriter w(buf, 0);
    for (int k = 0; k < p.sh_bits / 8; ++k) w.put(p.sh[k], 8);
    if (p.sh_bits & 7) w.put(p.sh[p.sh_bits / 8] >> (8 - (p.sh_bits & 7)), p.sh_bits & 7);
    w.flush();
  }
  BitWriter w(buf, mb_bits(p)[i]);
  const uint32_t run = mb_runs(p)[i];
  if (run != ~0u) put_ue(w, run);
  write_mb(w, p, m, i);
  w.flush();
}

// ---- 6. NAL unit: start codes, parameter sets, trailing bits, emulation prevention -----------------------------------

__global__ void __launch_bounds__(kFrameThreads) lspv_finish_kernel(const Params p) {
  const uint32_t total = mb_bits(p)[p.nmb];                      // RBSP bits before rbsp_trailing_bits
  const uint32_t nbytes = total / 8 + 1;
  const uint32_t* src = bit_buf(p);
  uint8_t* out = p.out;
  for (int i = threadIdx.x; i < p.ps_len; i += kFrameThreads) out[i] = p.ps[i];
  if (threadIdx.x == 0) {
    out[p.ps_len] = out[p.ps_len + 1] = out[p.ps_len + 2] = 0;
    out[p.ps_len + 3] = 1;
    out[p.ps_len + 4] = p.nal_header;
  }
  uint8_t* dst = out + p.ps_len + 5;
  auto byte_at = [&](uint32_t k) -> uint32_t {
    uint32_t b = (src[k >> 2] >> (24 - 8 * (k & 3))) & 255;
    if (k == total / 8) b |= 0x80u >> (total & 7);               // the stop bit
    return b;
  };
  // An 0x03 goes before byte k when k <= 3 and the run of zero bytes right before it has even length >= 2.
  int base = 0, last_nz = -1;
  for (uint32_t r0 = 0; r0 < nbytes; r0 += 8 * kFrameThreads) {
    const uint32_t at = r0 + 8 * threadIdx.x;
    uint32_t bytes[8];
    int mine = -1;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      bytes[i] = at + i < nbytes ? byte_at(at + i) : 1;
      if (at + i < nbytes && bytes[i]) mine = static_cast<int>(at + i);
    }
    int round_last;
    int prev_nz = max(last_nz, block_exclusive_scan<Max>(mine, &round_last));
    uint32_t count = 0;
    int nz = prev_nz;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (at + i >= nbytes) break;
      const int zeros = static_cast<int>(at + i) - nz - 1;
      count += 1 + (bytes[i] <= 3 && zeros >= 2 && !(zeros & 1));
      if (bytes[i]) nz = static_cast<int>(at + i);
    }
    int round_total;
    int o = base + block_exclusive_scan<Sum>(static_cast<int>(count), &round_total);
    nz = prev_nz;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (at + i >= nbytes) break;
      const int zeros = static_cast<int>(at + i) - nz - 1;
      if (bytes[i] <= 3 && zeros >= 2 && !(zeros & 1)) dst[o++] = 3;
      dst[o++] = static_cast<uint8_t>(bytes[i]);
      if (bytes[i]) nz = static_cast<int>(at + i);
    }
    base += round_total;
    last_nz = max(last_nz, round_last);
  }
  if (threadIdx.x == 0) {
    *p.size = p.ps_len + 5 + base;
    *p.is_idr = static_cast<uint8_t>(p.idr);
    *reinterpret_cast<int64_t*>(p.state) = p.frame + 1;
  }
}

// ---- host side ------------------------------------------------------------------------------------------------------

struct HostBits {
  std::string bits;
  void u(int n, uint32_t v) {
    for (int i = n - 1; i >= 0; --i) bits.push_back((v >> i) & 1 ? '1' : '0');
  }
  void ue(uint32_t v) {
    int k = 0;
    while ((v + 1) >> k) ++k;
    u(k - 1, 0);
    u(k, v + 1);
  }
  void se(int v) { ue(v > 0 ? 2u * v - 1 : 2u * static_cast<uint32_t>(-v)); }
  std::string rbsp() const {                                     // with rbsp_trailing_bits, as bytes
    std::string b = bits + "1";
    while (b.size() % 8) b.push_back('0');
    std::string out;
    for (size_t i = 0; i < b.size(); i += 8) {
      int v = 0;
      for (int k = 0; k < 8; ++k) v = 2 * v + (b[i + k] == '1');
      out.push_back(static_cast<char>(v));
    }
    return out;
  }
};

std::string nal_unit(int header, const std::string& rbsp) {
  std::string out("\0\0\0\1", 4);
  out.push_back(static_cast<char>(header));
  int zeros = 0;
  for (unsigned char b : rbsp) {
    if (zeros >= 2 && b <= 3) out.push_back(3), zeros = 0;
    out.push_back(static_cast<char>(b));
    zeros = b == 0 ? zeros + 1 : 0;
  }
  return out;
}

int level_idc_of(int height, int width, int fps) {
  const int64_t mbw = width / 16, mbh = height / 16, fs = mbw * mbh;
  for (const auto& l : kLevels)
    if (fs <= l[2] && mbw * mbw <= 8 * l[2] && mbh * mbh <= 8 * l[2] && fs * fps <= l[1] && fs <= l[3])
      return static_cast<int>(l[0]);
  return 0;
}

std::string parameter_sets(int height, int width, int fps) {
  HostBits s;
  s.u(8, 66), s.u(8, 0xC0), s.u(8, level_idc_of(height, width, fps));
  s.ue(0), s.ue(0), s.ue(2), s.ue(1), s.u(1, 0);
  s.ue(width / 16 - 1), s.ue(height / 16 - 1);
  s.u(1, 1), s.u(1, 1), s.u(1, 0);
  s.u(1, 1);                                                     // VUI
  s.u(1, 0), s.u(1, 0);
  s.u(1, 1), s.u(3, 5), s.u(1, 0), s.u(1, 1), s.u(8, 6), s.u(8, 6), s.u(8, 6);
  s.u(1, 0);
  s.u(1, 1), s.u(32, 1), s.u(32, 2 * fps), s.u(1, 1);
  s.u(1, 0), s.u(1, 0), s.u(1, 0);
  s.u(1, 1), s.u(1, 1), s.ue(0), s.ue(0), s.ue(16), s.ue(16), s.ue(0), s.ue(1);
  HostBits q;
  q.ue(0), q.ue(0), q.u(1, 0), q.u(1, 0), q.ue(0), q.ue(0), q.ue(0), q.u(1, 0), q.u(2, 0);
  q.se(0), q.se(0), q.se(0), q.u(1, 1), q.u(1, 0), q.u(1, 0);
  return nal_unit(0x67, s.rbsp()) + nal_unit(0x68, q.rbsp());
}

HostBits slice_header(int64_t frame, int gop, int qp) {
  const bool idr = frame % gop == 0;
  HostBits w;
  w.ue(0), w.ue(idr ? 7 : 5), w.ue(0), w.u(4, static_cast<uint32_t>((frame % gop) % 16));
  if (idr) w.ue(static_cast<uint32_t>((frame / gop) & 1));
  else w.u(1, 0), w.u(1, 0);
  if (idr) w.u(1, 0), w.u(1, 0);
  else w.u(1, 0);
  w.se(qp - 26);
  w.ue(1);
  return w;
}

int se_len(int v) {
  uint32_t k = v > 0 ? 2u * v - 1 : 2u * static_cast<uint32_t>(-v), n = 0;
  while ((k + 1) >> n) ++n;
  return static_cast<int>(2 * n - 1);
}

int64_t worst_block_bits(int n) { return n == 4 ? 8 + 4 * 28 + 3 + 3 * 2 : 16 + n * 28 + 9 + (n - 1) * 11; }

int64_t max_bytes_of(int height, int width) {
  const int64_t mbs = static_cast<int64_t>(height / 16) * (width / 16);
  const int64_t chroma = 2 * worst_block_bits(4) + 8 * worst_block_bits(15);
  const int64_t intra = 9 + 5 + 1 + worst_block_bits(16) + 16 * worst_block_bits(15) + chroma;
  const int64_t inter = 1 + 2 * se_len(-8 * kMaxSearch) + 11 + 1 + 16 * worst_block_bits(16) + chroma;
  int64_t run = 0;
  while ((mbs + 1) >> run) ++run;
  const int64_t mb = (intra > inter ? intra : inter) + 2 * run - 1;
  const int64_t rbsp = (64 + mbs * mb + 8 + 7) / 8;
  return 2 * 64 + 5 + rbsp + (rbsp + 1) / 2;
}

Layout layout_of(int height, int width) {
  const size_t hw = static_cast<size_t>(height) * width, nmb = hw / 256;
  const size_t words = static_cast<size_t>(max_bytes_of(height, width)) / 4 + 8;
  Layout l;
  l.yuv = 0;
  l.rec = align256(hw * 3 / 2);
  l.mbs = l.rec + align256(hw * 3 / 2);
  l.bits = l.mbs + align256(nmb * sizeof(MbRec));
  l.runs = l.bits + align256((nmb + 1) * sizeof(uint32_t));
  l.counters = l.runs + align256(nmb * sizeof(uint32_t));
  l.buf = l.counters + align256((height / 16 + 1) * sizeof(int));
  l.bytes = l.buf + align256(words * sizeof(uint32_t));
  return l;
}

int check_shape(int height, int width, int fps) {
  if (height < 16 || width < 16 || height > 65535 || width > 65535 || height % 16 || width % 16)
    return fail(LSPG_EINVAL, "height and width must be multiples of 16 in [16, 65535] (got %d x %d)", height, width);
  if (max_bytes_of(height, width) > kMaxAuBytes)
    return fail(LSPG_EINVAL, "a %d x %d frame has a worst-case access unit above the 2^30 bytes this encoder supports",
                height, width);
  if (level_idc_of(height, width, fps) == 0)
    return fail(LSPG_EINVAL, "no level of Table A-1 holds %d x %d at %d fps", height, width, fps);
  return LSPG_OK;
}

}  // namespace

struct lspv_ctx {
  int device = -1;
  int qp = 26, gop = 60, search = 16, fps = 60;
};

extern "C" {

const char* lspv_last_error(void) { return capi::last_error<Lspv>().c_str(); }

int lspv_destroy(lspv_handle h) {
  delete h;
  return LSPG_OK;
}

int lspv_create(lspv_handle* out, int qp, int gop, int search, int fps, int device) {
  if (!out) return fail(LSPG_EINVAL, "null argument");
  *out = nullptr;
  if (qp < 0 || qp > 51) return fail(LSPG_EINVAL, "qp must be in [0, 51] (got %d)", qp);
  if (gop < 1) return fail(LSPG_EINVAL, "gop must be >= 1 (got %d)", gop);
  if (search < 0 || search > kMaxSearch) return fail(LSPG_EINVAL, "search must be in [0, %d] (got %d)", kMaxSearch, search);
  if (fps < 1 || fps > 1000) return fail(LSPG_EINVAL, "fps must be in [1, 1000] (got %d)", fps);
  cudaDeviceProp prop;
  if (int rc = capi::check_device<Lspv>(device, &prop)) return rc;
  lspv_ctx* h = new lspv_ctx;
  h->device = device, h->qp = qp, h->gop = gop, h->search = search, h->fps = fps;
  *out = h;
  return LSPG_OK;
}

int lspv_max_bytes(lspv_handle h, int height, int width, size_t* bytes) {
  if (!h || !bytes) return fail(LSPG_EINVAL, "null argument");
  if (int rc = check_shape(height, width, h->fps)) return rc;
  *bytes = static_cast<size_t>(max_bytes_of(height, width));
  return LSPG_OK;
}

int lspv_state_bytes(lspv_handle h, int height, int width, size_t* bytes) {
  if (!h || !bytes) return fail(LSPG_EINVAL, "null argument");
  if (int rc = check_shape(height, width, h->fps)) return rc;
  *bytes = kStateHeader + static_cast<size_t>(height) * width * 3 / 2;
  return LSPG_OK;
}

int lspv_workspace_bytes(lspv_handle h, int height, int width, size_t* bytes) {
  if (!h || !bytes) return fail(LSPG_EINVAL, "null argument");
  if (int rc = check_shape(height, width, h->fps)) return rc;
  *bytes = layout_of(height, width).bytes;
  return LSPG_OK;
}

int lspv_encode(lspv_handle h, const uint8_t* images, int n, int height, int width, int components, int64_t f0,
                void* state, uint8_t* out, int64_t out_stride, int32_t* sizes, uint8_t* is_idr, void* ws,
                size_t ws_bytes, void* stream) {
  if (!h) return fail(LSPG_EINVAL, "null handle");
  if (n < 0) return fail(LSPG_EINVAL, "n must be >= 0 (got %d)", n);
  if (f0 < 0) return fail(LSPG_EINVAL, "f0 must be >= 0 (got %lld)", static_cast<long long>(f0));
  if (components != 1 && components != 3) return fail(LSPG_EINVAL, "components must be 1 or 3 (got %d)", components);
  if (int rc = check_shape(height, width, h->fps)) return rc;
  const int64_t bound = max_bytes_of(height, width);
  if (out_stride < bound)
    return fail(LSPG_EINVAL, "out_stride must be at least lspv_max_bytes = %lld (got %lld)", static_cast<long long>(bound),
                static_cast<long long>(out_stride));
  const Layout lay = layout_of(height, width);
  if (ws_bytes < lay.bytes)
    return fail(LSPG_EINVAL, "workspace of %zu bytes is smaller than lspv_workspace_bytes = %zu", ws_bytes, lay.bytes);
  if (n > 0 && (!images || !state || !out || !sizes || !is_idr || !ws)) return fail(LSPG_EINVAL, "null buffer");
  if (reinterpret_cast<uintptr_t>(ws) % 256 || reinterpret_cast<uintptr_t>(state) % 256)
    return fail(LSPG_EINVAL, "ws and state must be 256-byte aligned");
  if (int rc = capi::require_device<Lspv>(h->device, "lspv_encode")) return rc;
  if (n == 0) return LSPG_OK;
  DeviceGuard g(h->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const std::string ps = parameter_sets(height, width, h->fps);
  const int span = 16 + 2 * h->search, pitch = (span + 3) / 4 + 1;
  const size_t win_bytes = static_cast<size_t>(span) * pitch * 4;      // at most 21 KB (search 64)
  Params p;
  std::memset(&p, 0, sizeof(p));
  p.ws = static_cast<uint8_t*>(ws);
  p.state = static_cast<uint8_t*>(state);
  p.lay = lay;
  p.height = height, p.width = width, p.comps = components;
  p.mbw = width / 16, p.mbh = height / 16, p.nmb = p.mbw * p.mbh;
  p.qp = h->qp, p.search = h->search;
  const size_t frame_bytes = static_cast<size_t>(height) * width * components;
  const size_t yuv_bytes = static_cast<size_t>(height) * width * 3 / 2;
  const int colour_blocks = (height / 2 * (width / 2) + kThreads - 1) / kThreads;
  for (int i = 0; i < n; ++i) {
    const int64_t f = f0 + i;
    p.image = images + i * frame_bytes;
    p.out = out + i * out_stride;
    p.size = sizes + i;
    p.is_idr = is_idr + i;
    p.frame = f;
    p.idr = f % h->gop == 0;
    p.ps_len = p.idr ? static_cast<int>(ps.size()) : 0;
    if (p.idr) std::memcpy(p.ps, ps.data(), ps.size());
    const HostBits sh = slice_header(f, h->gop, h->qp);
    p.sh_bits = static_cast<int>(sh.bits.size());
    std::memset(p.sh, 0, sizeof(p.sh));
    for (int k = 0; k < p.sh_bits; ++k)
      if (sh.bits[k] == '1') p.sh[k / 8] |= 0x80 >> (k % 8);
    p.nal_header = p.idr ? 0x65 : 0x61;
    lspv_colour_kernel<<<colour_blocks, kThreads, 0, s>>>(p);
    if (p.idr) {
      CUDA_TRY(cudaMemsetAsync(p.ws + lay.counters, 0, (p.mbh + 1) * sizeof(int), s));
      lspv_intra_kernel<<<p.mbh, kThreads, 0, s>>>(p);
    } else {
      lspv_inter_kernel<<<dim3(p.mbw, p.mbh), kThreads, win_bytes, s>>>(p);
    }
    lspv_bits_kernel<<<(p.nmb + 127) / 128, 128, 0, s>>>(p);
    lspv_offsets_kernel<<<1, kFrameThreads, 0, s>>>(p);
    lspv_pack_kernel<<<(p.nmb + 127) / 128, 128, 0, s>>>(p);
    lspv_finish_kernel<<<1, kFrameThreads, 0, s>>>(p);
    CUDA_TRY(cudaMemcpyAsync(p.state + kStateHeader, p.ws + lay.rec, yuv_bytes, cudaMemcpyDeviceToDevice, s));
  }
  CUDA_TRY(cudaGetLastError());
  return LSPG_OK;
}

}  // extern "C"
