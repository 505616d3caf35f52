// C-ABI implementation of the log-mel front end (see include/lspa.h; SURVEY.md 8f row N6).
//
// Reference: funcs/utils.py compute_mel_one_sequence (:61-83) loops over 2 nframe windows in Python; each window is one
// Audio2Mel.forward call (funcs/audio_funcs.py:56-75) on a 266-sample clip: F.pad(reflect, 189), torch.stft(n_fft 512,
// win_length 266, center=False) -> exactly one frame, sqrt(re^2 + im^2), mel_basis @ magnitude, log(clamp(., 1e-5)),
// (x - m) / -m.
//
// Here one launch of lspa_logmel_kernel computes every window.  One CTA of 256 threads owns kWin = 16 consecutive
// windows:
//   1. frame: the 266 nonzero taps of each windowed frame, hann[t] * clip[reflect(t - 66)], built from the audio in
//      global memory (read-only cache; consecutive windows overlap by ~133 samples) into shared memory [t][window].
//   2. DFT: thread k < 256 computes bin k of all 16 windows as a direct real DFT over the 266 taps, in tap order, with
//      one fma per (tap, window) into re and im; the twiddle of tap t is cos/sin(2 pi (k (t + 123) mod 512) / 512) from a
//      512-entry float2 table in shared memory (built in fp64 on the host and rounded once, so the argument reduction
//      is exact).  The index advances by k per tap.  Bin 256 (twiddle +-1) is a signed sum, 16 lanes per window.
//   3. magnitude sqrt(re*re + im*im) in fp32 to shared memory; then thread (m, half) sums basis[m][k] * mag[k] over k in
//      order for 8 windows (the basis is read through the read-only cache: 82 KB in shared memory would cap the SM at
//      two CTAs, and every CTA reads it once either way), takes logf(max(., 1e-5f)) and normalises in fp32 as torch
//      does ((x - m) / -m with m rounded to fp32, an IEEE division).
//   4. the CTA's [16, n_mels] block is staged in shared memory and stored with consecutive addresses.
// No atomics and a fixed summation order everywhere: results are bit-identical from run to run.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <string>

#include "../../include/lspa.h"

namespace {

thread_local std::string g_aerr;

int afail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_aerr = buf;
  return code;
}

#define ACUDA_TRY(expr)                                                                           \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) return afail(LSPG_ECUDA, "%s failed: %s", #expr, cudaGetErrorString(_e)); \
  } while (0)

constexpr int kNfft = 512;
constexpr int kBins = kNfft / 2 + 1;           // 257
constexpr int kWinLen = 266;                   // Audio2Mel's win_length: the Hann window, whatever the clip length
constexpr int kHop = 133;
constexpr int kPad = (kNfft - kHop) / 2;       // 189: reflect pad on each side of the clip
constexpr int kWinOff = (kNfft - kWinLen) / 2; // 123: the window's place in the 512-sample frame
constexpr int kMinFrame = kPad + 1, kMaxFrame = kWinLen;
constexpr int kMaxMels = 128;
constexpr int kWin = 16;                       // windows per CTA
constexpr int kThreads = 256;
constexpr unsigned kFull = 0xffffffffu;

struct Smem {
  float frame[kWinLen][kWin];                  // windowed taps; reused as the [kWin][n_mels] output stage
  float mag[kBins][kWin];
  float2 tw[kNfft];                            // (cos, sin) of 2 pi j / 512
  float hann[kWinLen];
};
static_assert(kWin * kMaxMels <= kWinLen * kWin, "output stage must fit in the frame buffer");
static_assert(2 * kMaxMels <= kThreads, "one thread per (mel, half of the windows)");

__global__ void __launch_bounds__(kThreads) lspa_logmel_kernel(const float* __restrict__ audio, int64_t n_samples,
                                                               int n_windows, int frame_len, double step,
                                                               const float2* __restrict__ tw_g, const float* __restrict__ hann_g,
                                                               const float* __restrict__ basis, int n_mels, int normalize,
                                                               float* __restrict__ out) {
  __shared__ __align__(16) Smem sm;
  const int tid = threadIdx.x;
  const int w0 = blockIdx.x * kWin;
  const int nw = min(kWin, n_windows - w0);
  for (int j = tid; j < kNfft; j += kThreads) sm.tw[j] = tw_g[j];
  for (int j = tid; j < kWinLen; j += kThreads) sm.hann[j] = hann_g[j];
  __syncthreads();

  // 1. frame[t][g] = hann[t] * clip_g[p], p the reflect-padded clip position of frame sample t + 123
  for (int e = tid; e < kWinLen * kWin; e += kThreads) {
    const int t = e / kWin, g = e % kWin;
    float v = 0.f;
    if (g < nw) {
      const int64_t st = static_cast<int64_t>(__dmul_rn(static_cast<double>(w0 + g), step));
      int p = t + kWinOff - kPad;
      if (p < 0) p = -p;
      if (p >= frame_len) p = 2 * (frame_len - 1) - p;
      const int64_t a = st + p;
      if (a < n_samples) v = __fmul_rn(sm.hann[t], __ldg(audio + a));
    }
    sm.frame[t][g] = v;
  }
  __syncthreads();

  // 2. bins 0..255: thread k; the twiddle index k (t + 123) mod 512 advances by k per tap
  {
    const int k = tid;
    float re[kWin], im[kWin];
#pragma unroll
    for (int g = 0; g < kWin; ++g) re[g] = im[g] = 0.f;
    int j = (k * kWinOff) & (kNfft - 1);
#pragma unroll 2
    for (int t = 0; t < kWinLen; ++t) {
      const float2 c = sm.tw[j];
      j = (j + k) & (kNfft - 1);
      const float4* x4 = reinterpret_cast<const float4*>(sm.frame[t]);
#pragma unroll
      for (int q = 0; q < kWin / 4; ++q) {
        const float4 x = x4[q];
        re[4 * q + 0] = fmaf(x.x, c.x, re[4 * q + 0]); im[4 * q + 0] = fmaf(x.x, c.y, im[4 * q + 0]);
        re[4 * q + 1] = fmaf(x.y, c.x, re[4 * q + 1]); im[4 * q + 1] = fmaf(x.y, c.y, im[4 * q + 1]);
        re[4 * q + 2] = fmaf(x.z, c.x, re[4 * q + 2]); im[4 * q + 2] = fmaf(x.z, c.y, im[4 * q + 2]);
        re[4 * q + 3] = fmaf(x.w, c.x, re[4 * q + 3]); im[4 * q + 3] = fmaf(x.w, c.y, im[4 * q + 3]);
      }
    }
#pragma unroll
    for (int g = 0; g < kWin; ++g) sm.mag[k][g] = __fsqrt_rn(__fadd_rn(__fmul_rn(re[g], re[g]), __fmul_rn(im[g], im[g])));
  }
  // bin 256: sum_t (-1)^(t + 123) frame[t], lane l of each 16-lane group takes the taps t = l mod 16
  {
    const int g = tid >> 4, l = tid & 15;
    float s = 0.f;
    for (int t = l; t < kWinLen; t += 16) s += ((t + kWinOff) & 1) ? -sm.frame[t][g] : sm.frame[t][g];
#pragma unroll
    for (int off = 8; off; off >>= 1) s += __shfl_xor_sync(kFull, s, off);
    if (l == 0) sm.mag[kBins - 1][g] = fabsf(s);
  }
  __syncthreads();

  // 3. mel, log, normalise: thread (m, half) -> windows half*8 .. half*8+7; results staged in the frame buffer
  float* stage = &sm.frame[0][0];
  if (tid < 2 * n_mels) {
    const int m = tid >> 1, h = (tid & 1) * (kWin / 2);
    const float* b = basis + static_cast<size_t>(m) * kBins;
    float acc[kWin / 2];
#pragma unroll
    for (int g = 0; g < kWin / 2; ++g) acc[g] = 0.f;
    for (int k = 0; k < kBins; ++k) {
      const float bk = __ldg(b + k);
      const float4 x0 = *reinterpret_cast<const float4*>(&sm.mag[k][h]);
      const float4 x1 = *reinterpret_cast<const float4*>(&sm.mag[k][h + 4]);
      acc[0] = fmaf(bk, x0.x, acc[0]); acc[1] = fmaf(bk, x0.y, acc[1]);
      acc[2] = fmaf(bk, x0.z, acc[2]); acc[3] = fmaf(bk, x0.w, acc[3]);
      acc[4] = fmaf(bk, x1.x, acc[4]); acc[5] = fmaf(bk, x1.y, acc[5]);
      acc[6] = fmaf(bk, x1.z, acc[6]); acc[7] = fmaf(bk, x1.w, acc[7]);
    }
    constexpr float mmin = static_cast<float>(-11.512925464970229);   // log(1e-5) rounded to fp32, as torch rounds it
#pragma unroll
    for (int g = 0; g < kWin / 2; ++g) {
      float v = logf(fmaxf(acc[g], 1e-5f));
      if (normalize) v = __fdiv_rn(__fsub_rn(v, mmin), -mmin);
      stage[(h + g) * n_mels + m] = v;
    }
  }
  __syncthreads();

  // 4. the CTA's rows are contiguous in out
  float* dst = out + static_cast<int64_t>(w0) * n_mels;
  for (int e = tid; e < nw * n_mels; e += kThreads) dst[e] = stage[e];
}

class DeviceGuard {
 public:
  explicit DeviceGuard(int dev) { cudaGetDevice(&prev_); if (prev_ != dev) cudaSetDevice(dev); dev_ = dev; }
  ~DeviceGuard() { if (prev_ != dev_) cudaSetDevice(prev_); }
 private:
  int prev_ = 0, dev_ = 0;
};

}  // namespace

struct lspa_ctx {
  int device = -1;
  int n_mels = 0;              // 0 until a basis is loaded
  float2* d_tw = nullptr;
  float* d_hann = nullptr;
  float* d_basis = nullptr;    // [kMaxMels, kBins]
};

extern "C" {

const char* lspa_last_error(void) { return g_aerr.c_str(); }

int lspa_destroy(lspa_handle h) {
  if (!h) return LSPG_OK;
  if (h->device >= 0) {
    DeviceGuard g(h->device);
    if (h->d_tw) cudaFree(h->d_tw);
    if (h->d_hann) cudaFree(h->d_hann);
    if (h->d_basis) cudaFree(h->d_basis);
  }
  delete h;
  return LSPG_OK;
}

int lspa_create(lspa_handle* out, int device) {
  if (!out) return afail(LSPG_EINVAL, "null argument");
  *out = nullptr;
  if (device < -1) return afail(LSPG_EINVAL, "device must be >= -1 (got %d)", device);
  if (device >= 0) {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) return afail(LSPG_ENODEV, "no CUDA device: %s", cudaGetErrorString(e));
    if (device >= count) return afail(LSPG_ENODEV, "device %d out of range (%d devices)", device, count);
    cudaDeviceProp prop;
    ACUDA_TRY(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
      return afail(LSPG_ENODEV, "device %d is sm_%d%d; this library contains sm_90a code only (no fallback)", device, prop.major, prop.minor);
  }
  lspa_ctx* h = new lspa_ctx;
  h->device = device;
  if (device >= 0) {
    // twiddles cos/sin(2 pi j / 512) and the periodic Hann window 0.5 - 0.5 cos(2 pi t / 266), in fp64, rounded once
    float2 tw[kNfft];
    float hann[kWinLen];
    const double pi = 3.14159265358979323846;
    for (int j = 0; j < kNfft; ++j)
      tw[j] = make_float2(static_cast<float>(std::cos(2.0 * pi * j / kNfft)), static_cast<float>(std::sin(2.0 * pi * j / kNfft)));
    for (int t = 0; t < kWinLen; ++t) hann[t] = static_cast<float>(0.5 - 0.5 * std::cos(2.0 * pi * t / kWinLen));
    DeviceGuard g(device);
    cudaError_t e = cudaMalloc(&h->d_tw, sizeof(tw));
    if (e == cudaSuccess) e = cudaMalloc(&h->d_hann, sizeof(hann));
    if (e == cudaSuccess) e = cudaMalloc(&h->d_basis, sizeof(float) * kMaxMels * kBins);
    if (e == cudaSuccess) e = cudaMemcpy(h->d_tw, tw, sizeof(tw), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(h->d_hann, hann, sizeof(hann), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
      lspa_destroy(h);
      return afail(LSPG_ECUDA, "lspa_create: %s", cudaGetErrorString(e));
    }
  }
  *out = h;
  return LSPG_OK;
}

int lspa_load_mel_basis(lspa_handle h, const float* host_basis, int n_mels, int n_bins) {
  if (!h || !host_basis) return afail(LSPG_EINVAL, "null argument");
  if (n_mels < 1 || n_mels > kMaxMels) return afail(LSPG_EINVAL, "n_mels must be in [1, %d] (got %d)", kMaxMels, n_mels);
  if (n_bins != kBins) return afail(LSPG_EINVAL, "the basis must have %d columns (n_fft 512; got %d)", kBins, n_bins);
  if (h->device < 0) return afail(LSPG_ENODEV, "host-only handle: lspa_load_mel_basis needs an sm_90 device (no CPU path exists)");
  DeviceGuard g(h->device);
  h->n_mels = 0;                               // not usable until the copy is complete
  ACUDA_TRY(cudaMemcpy(h->d_basis, host_basis, sizeof(float) * n_mels * kBins, cudaMemcpyHostToDevice));
  h->n_mels = n_mels;
  return LSPG_OK;
}

int lspa_logmel(lspa_handle h, const float* audio, int64_t n_samples, int n_windows, int frame_len, double step,
                int normalize, float* out, void* stream) {
  if (!h) return afail(LSPG_EINVAL, "null handle");
  if (n_samples < 0) return afail(LSPG_EINVAL, "n_samples must be >= 0 (got %lld)", static_cast<long long>(n_samples));
  if (n_windows < 0) return afail(LSPG_EINVAL, "n_windows must be >= 0 (got %d)", n_windows);
  if (frame_len < kMinFrame || frame_len > kMaxFrame)
    return afail(LSPG_EINVAL, "frame_len must be in [%d, %d] (got %d): the reflect pad of %d needs a longer clip and one stft "
                 "frame a shorter one", kMinFrame, kMaxFrame, frame_len, kPad);
  if (!(step >= 0.0) || !(step * static_cast<double>(n_windows) < 4.0e18))
    return afail(LSPG_EINVAL, "step must be finite and >= 0, with n_windows * step < 4e18 (got %g)", step);
  if ((!audio && n_samples > 0) || (!out && n_windows > 0)) return afail(LSPG_EINVAL, "null buffer");
  if (h->device < 0) return afail(LSPG_ENODEV, "host-only handle: lspa_logmel needs an sm_90 device (no CPU path exists)");
  if (h->n_mels == 0) return afail(LSPG_ESTATE, "lspa_load_mel_basis has not been called");
  if (n_windows == 0) return LSPG_OK;
  DeviceGuard g(h->device);
  const int blocks = n_windows / kWin + (n_windows % kWin != 0);   // w0 = blockIdx.x * kWin < n_windows < 2^31
  lspa_logmel_kernel<<<blocks, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      audio, n_samples, n_windows, frame_len, step, h->d_tw, h->d_hann, h->d_basis, h->n_mels, normalize ? 1 : 0, out);
  ACUDA_TRY(cudaGetLastError());
  return LSPG_OK;
}

}  // extern "C"
