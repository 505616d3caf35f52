// Device code shared by the variable-length coders (lspj's Huffman coding, lspv's CAVLC).  Each item (a block, a
// macroblock) first counts its bits; one CTA per frame turns the counts into bit offsets with a block-wide scan; then one
// thread per item writes its codes at its offset.  A word can straddle two items, so words are written with atomicOr into
// a zeroed buffer: order-free, so the bytes do not vary from run to run.
#pragma once

#include <cstdint>

namespace bitstream {

// MSB-first codes into 32-bit words from bit `bit` of buf on.  put's precondition: size <= 32 and code < 2^size.
struct BitWriter {
  uint32_t* buf;
  uint32_t word;                // next word to write
  int n;                        // bits held in acc (< 32 between puts)
  uint64_t acc;

  __device__ __forceinline__ BitWriter(uint32_t* b, uint32_t bit) : buf(b), word(bit >> 5), n(bit & 31), acc(0) {}

  __device__ __forceinline__ void put(uint32_t code, int size) {
    acc = (acc << size) | code;
    n += size;
    if (n >= 32) {
      n -= 32;
      atomicOr(buf + word++, static_cast<uint32_t>(acc >> n));
      acc &= (uint64_t(1) << n) - 1;
    }
  }
  __device__ __forceinline__ void flush() {
    if (n > 0) atomicOr(buf + word, static_cast<uint32_t>(acc << (32 - n)));
  }
};

struct Sum {
  static constexpr int kIdentity = 0;
  template <class T>
  __device__ __forceinline__ T operator()(T a, T b) const { return a + b; }
};
// The max of indices, -1 standing for none.
struct Max {
  static constexpr int kIdentity = -1;
  template <class T>
  __device__ __forceinline__ T operator()(T a, T b) const { return max(a, b); }
};

// The exclusive Op-scan of v over the CTA's threads in order, and in *total the reduction of all of them.  blockDim.x is a
// multiple of 32.  Ends with a barrier, so a kernel may call it again.
template <class Op, class T>
__device__ __forceinline__ T block_exclusive_scan(T v, T* total) {
  __shared__ T warp_acc[32];
  const Op op{};
  const T ident = static_cast<T>(Op::kIdentity);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  T incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl = op(incl, u);
  }
  if (lane == 31) warp_acc[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    T s = lane < nw ? warp_acc[lane] : ident;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const T u = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s = op(s, u);
    }
    if (lane < nw) warp_acc[lane] = s;
  }
  __syncthreads();
  T excl = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) excl = ident;
  if (wid) excl = op(warp_acc[wid - 1], excl);
  *total = warp_acc[nw - 1];
  __syncthreads();
  return excl;
}

// The items [i0, i1) of n that thread threadIdx.x takes in a CTA-wide pass: consecutive runs in thread order, so one
// scan over the threads orders all items.
struct Chunk {
  int i0, i1;
  __device__ __forceinline__ explicit Chunk(int n) {
    const int per = (n + blockDim.x - 1) / blockDim.x;
    i0 = min(n, static_cast<int>(threadIdx.x) * per);
    i1 = min(n, i0 + per);
  }
};

// Called by the whole CTA: adds extra(i) to each bit count bits[i], i < n, then rewrites the counts in place as the
// items' first bits, base plus the sum of the counts before; stores the end (base plus all counts) at bits[n] and
// returns it.  Each thread calls extra once per item of its Chunk(n), in increasing order, in the pass that sums the
// counts, so no count is stored and loaded back before the scan.  T is the type the sums are formed in.
template <class T, class Extra>
__device__ __forceinline__ T counts_to_offsets(uint32_t* bits, int n, T base, Extra extra) {
  const Chunk c(n);
  T sum = 0;
  for (int i = c.i0; i < c.i1; ++i) {
    const T b = static_cast<T>(bits[i]) + extra(i);
    bits[i] = static_cast<uint32_t>(b);
    sum += b;
  }
  T total;
  T at = base + block_exclusive_scan<Sum>(sum, &total);
  for (int i = c.i0; i < c.i1; ++i) {
    const T b = static_cast<T>(bits[i]);
    bits[i] = static_cast<uint32_t>(at);
    at += b;
  }
  total += base;
  if (threadIdx.x == 0) bits[n] = static_cast<uint32_t>(total);
  return total;
}

}  // namespace bitstream
