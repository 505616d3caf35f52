// fp32 GEMM for the hoisted (non-recurrent) parts of the audio networks, shared by csrc/lsph.cu and csrc/lspr.cu:
//   C[M,N] = epilogue( A[M,K] * W[N,K]^T ),  epilogue v -> v*scale[n] + shift[n], then LeakyReLU(0.2) if `leaky`.
// 64x64 tile, K step 16, 256 threads x (4x4) outputs, every output summed over k in increasing order with fmaf.
// K % 16 == 0, rows of A and W 16-byte aligned, M ragged.  N % 64 == 0 unless kRaggedN (rows of W past N read as zero,
// columns past N not stored).  The template flag only changes which addresses are read; the arithmetic of every
// instantiation is the same.
#pragma once

#include <cuda_runtime.h>

#include <cstddef>

template <bool kRaggedN = false>
__global__ void __launch_bounds__(256) gemm_nt_kernel(const float* __restrict__ A, const float* __restrict__ W,
                                                      const float* __restrict__ scale, const float* __restrict__ shift,
                                                      float* __restrict__ C, int M, int N, int K, int leaky) {
  __shared__ float As[16][64 + 4];
  __shared__ float Ws[16][64 + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  float acc[4][4] = {};
  const int lr = threadIdx.x >> 2;            // 0..63: tile row loaded by this thread
  const int lk = (threadIdx.x & 3) * 4;       // 0,4,8,12: first of its 4 k values
  for (int k0 = 0; k0 < K; k0 += 16) {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m0 + lr < M) a = *reinterpret_cast<const float4*>(A + static_cast<size_t>(m0 + lr) * K + k0 + lk);
    float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!kRaggedN || n0 + lr < N) w = *reinterpret_cast<const float4*>(W + static_cast<size_t>(n0 + lr) * K + k0 + lk);
    As[lk + 0][lr] = a.x; As[lk + 1][lr] = a.y; As[lk + 2][lr] = a.z; As[lk + 3][lr] = a.w;
    Ws[lk + 0][lr] = w.x; Ws[lk + 1][lr] = w.y; Ws[lk + 2][lr] = w.z; Ws[lk + 3][lr] = w.w;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      float av[4], wv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { av[i] = As[k][ty * 4 + i]; wv[i] = Ws[k][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (kRaggedN && n >= N) continue;
      float v = fmaf(acc[i][j], scale[n], shift[n]);
      if (leaky) v = v > 0.f ? v : 0.2f * v;
      C[static_cast<size_t>(m) * N + n] = v;
    }
  }
}
