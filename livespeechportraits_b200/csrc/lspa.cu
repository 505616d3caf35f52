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

#include <algorithm>
#include <cmath>

#include "../../include/lspa.h"
#include "capi.cuh"

using capi::DeviceGuard;

namespace {

struct Lspa;
constexpr auto fail = capi::fail<Lspa>;

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

// audio holds clip samples [first_sample, first_sample + n_samples); samples past its end read as zero (the clip's end
// padding).  Block b computes windows first_window + b*kWin ..., stored from out row b*kWin.
__global__ void __launch_bounds__(kThreads) lspa_logmel_kernel(const float* __restrict__ audio, int64_t first_sample,
                                                               int64_t n_samples, int first_window, int n_windows,
                                                               int frame_len, double step,
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
      const int64_t st = static_cast<int64_t>(__dmul_rn(static_cast<double>(first_window + w0 + g), step));
      int p = t + kWinOff - kPad;
      if (p < 0) p = -p;
      if (p >= frame_len) p = 2 * (frame_len - 1) - p;
      const int64_t a = st + p - first_sample;
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

// ---------------------------------------------------------------------------------------------------------------------
// librosa.load's resampling (resampy.resample_f with a kaiser table): one thread per output sample.
//
// The time register of output t is the reference's running fp64 sum 0 + 1/r + 1/r + ..., evaluated from a host table
// of its closed form per binade: rows t_b, base, k, e with register(t) = (base + (t - t_b) k) 2^e for t_b <= t < the
// next row's t_b.  The int64 product is exact (< 2^53) and the scaling by 2^e is exact, so the value is the serial
// sum's bits.  Each tap is the reference's fp64 expression, weight = win[j] + eta delta[j], y = fp32(y + weight x), with
// explicit _rn intrinsics so that nvcc contracts nothing into a DFMA.  Inputs before sample 0 or outside the buffer read
// as +0, which leaves y unchanged: the same bits as the reference's wing clamps.
constexpr int kRsThreads = 256;
constexpr int kMaxRegRows = 64;                // register rows per launch; a span over more rows is split

struct RegRows {
  int n;
  int64_t t0[kMaxRegRows], base[kMaxRegRows], k[kMaxRegRows];
  int e[kMaxRegRows];
};

__device__ __forceinline__ double pow2(int e) { return __longlong_as_double(static_cast<long long>(e + 1023) << 52); }

// Frame j of the buffer (clip frame first_in + j) decoded as soundfile does and mixed to mono as librosa's to_mono.
template <int FMT, int CH>
__device__ __forceinline__ float mono_at(const void* frames, int64_t j) {
  float c[CH];
#pragma unroll
  for (int q = 0; q < CH; ++q) {
    if (FMT == LSPA_FMT_S16)
      c[q] = __fmul_rn(static_cast<float>(__ldg(static_cast<const short*>(frames) + j * CH + q)), 1.0f / 32768.0f);
    else
      c[q] = __ldg(static_cast<const float*>(frames) + j * CH + q);
  }
  return CH == 1 ? c[0] : __fmul_rn(__fadd_rn(c[0], c[CH - 1]), 0.5f);
}

// One wing: n_taps taps from table entry `offset` in steps of index_step, input frames p0, p0 + dir, ...
template <int FMT, int CH>
__device__ __forceinline__ float wing(float y, const double2* __restrict__ tab, int offset, int index_step, int n_taps,
                                      double eta, const void* frames, int64_t p0, int dir, int64_t n_in) {
#pragma unroll 4
  for (int i = 0; i < n_taps; ++i) {
    const double2 wd = __ldg(tab + offset + i * index_step);                 // (win, delta)
    const double weight = __dadd_rn(wd.x, __dmul_rn(eta, wd.y));
    const int64_t p = p0 + static_cast<int64_t>(dir) * i;
    const float x = (p >= 0 && p < n_in) ? mono_at<FMT, CH>(frames, p) : 0.0f;
    y = __double2float_rn(__dadd_rn(static_cast<double>(y), __dmul_rn(weight, static_cast<double>(x))));
  }
  return y;
}

// Outputs first_out .. first_out + n_out - 1 into out[0 ..]; frames holds clip frames [first_in, first_in + n_in).
template <int FMT, int CH>
__global__ void __launch_bounds__(kRsThreads) lspa_resample_kernel(const void* __restrict__ frames, int64_t first_in,
                                                                   int64_t n_in, int64_t first_out, int64_t n_out,
                                                                   RegRows reg, const double2* __restrict__ tab,
                                                                   int nwin, int num_table, int index_step, double scale,
                                                                   float* __restrict__ out) {
  const int64_t o = static_cast<int64_t>(blockIdx.x) * kRsThreads + threadIdx.x;
  if (o >= n_out) return;
  const int64_t t = first_out + o;
  int r = 0;                                   // the last row with t0 <= t
  for (int s = kMaxRegRows / 2; s; s >>= 1)
    if (r + s < reg.n && reg.t0[r + s] <= t) r += s;
  const double tr = __dmul_rn(static_cast<double>(reg.base[r] + (t - reg.t0[r]) * reg.k[r]), pow2(reg.e[r]));
  const int64_t n = static_cast<int64_t>(tr);
  const double dn = static_cast<double>(n);
  const double frac = __dmul_rn(scale, __dsub_rn(tr, dn));
  double index_frac = __dmul_rn(frac, static_cast<double>(num_table));
  int offset = static_cast<int>(index_frac);
  double eta = __dsub_rn(index_frac, static_cast<double>(offset));
  float y = wing<FMT, CH>(0.0f, tab, offset, index_step, (nwin - offset) / index_step, eta, frames, n - first_in, -1, n_in);
  index_frac = __dmul_rn(__dsub_rn(scale, frac), static_cast<double>(num_table));
  offset = static_cast<int>(index_frac);
  eta = __dsub_rn(index_frac, static_cast<double>(offset));
  y = wing<FMT, CH>(y, tab, offset, index_step, (nwin - offset) / index_step, eta, frames, n + 1 - first_in, 1, n_in);
  out[o] = y;
}

}  // namespace

struct lspa_ctx {
  int device = -1;
  int n_mels = 0;              // 0 until a basis is loaded
  float2* d_tw = nullptr;
  float* d_hann = nullptr;
  float* d_basis = nullptr;    // [kMaxMels, kBins]
  // the resampling filter: 0 entries until one is loaded
  int nwin = 0, num_table = 0, index_step = 0;
  double scale = 0.0;
  double2* d_rs_tab = nullptr; // [nwin] (win, delta)
};

extern "C" {

const char* lspa_last_error(void) { return capi::last_error<Lspa>().c_str(); }

int lspa_destroy(lspa_handle h) {
  if (!h) return LSPG_OK;
  if (h->device >= 0) {
    DeviceGuard g(h->device);
    if (h->d_tw) cudaFree(h->d_tw);
    if (h->d_hann) cudaFree(h->d_hann);
    if (h->d_basis) cudaFree(h->d_basis);
    if (h->d_rs_tab) cudaFree(h->d_rs_tab);
  }
  delete h;
  return LSPG_OK;
}

int lspa_create(lspa_handle* out, int device) {
  if (!out) return fail(LSPG_EINVAL, "null argument");
  *out = nullptr;
  cudaDeviceProp prop;
  if (int rc = capi::check_device<Lspa>(device, &prop)) return rc;
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
      return fail(LSPG_ECUDA, "lspa_create: %s", cudaGetErrorString(e));
    }
  }
  *out = h;
  return LSPG_OK;
}

int lspa_load_mel_basis(lspa_handle h, const float* host_basis, int n_mels, int n_bins) {
  if (!h || !host_basis) return fail(LSPG_EINVAL, "null argument");
  if (n_mels < 1 || n_mels > kMaxMels) return fail(LSPG_EINVAL, "n_mels must be in [1, %d] (got %d)", kMaxMels, n_mels);
  if (n_bins != kBins) return fail(LSPG_EINVAL, "the basis must have %d columns (n_fft 512; got %d)", kBins, n_bins);
  if (int rc = capi::require_device<Lspa>(h->device, "lspa_load_mel_basis")) return rc;
  DeviceGuard g(h->device);
  h->n_mels = 0;                               // not usable until the copy is complete
  CUDA_TRY(cudaMemcpy(h->d_basis, host_basis, sizeof(float) * n_mels * kBins, cudaMemcpyHostToDevice));
  h->n_mels = n_mels;
  return LSPG_OK;
}

int lspa_logmel_at(lspa_handle h, const float* audio, int64_t first_sample, int64_t n_samples, int first_window,
                   int n_windows, int frame_len, double step, int normalize, float* out, void* stream) {
  if (!h) return fail(LSPG_EINVAL, "null handle");
  if (n_samples < 0) return fail(LSPG_EINVAL, "n_samples must be >= 0 (got %lld)", static_cast<long long>(n_samples));
  if (n_windows < 0) return fail(LSPG_EINVAL, "n_windows must be >= 0 (got %d)", n_windows);
  if (frame_len < kMinFrame || frame_len > kMaxFrame)
    return fail(LSPG_EINVAL, "frame_len must be in [%d, %d] (got %d): the reflect pad of %d needs a longer clip and one stft "
                 "frame a shorter one", kMinFrame, kMaxFrame, frame_len, kPad);
  if (!(step >= 0.0) || !(step * (static_cast<double>(first_window) + n_windows) < 4.0e18))
    return fail(LSPG_EINVAL, "step must be finite and >= 0, with n_windows * step < 4e18 (got %g)", step);
  if ((!audio && n_samples > 0) || (!out && n_windows > 0)) return fail(LSPG_EINVAL, "null buffer");
  if (first_sample < 0 || first_window < 0 || static_cast<int64_t>(first_window) + n_windows > INT32_MAX)
    return fail(LSPG_EINVAL, "first_sample and first_window must be >= 0, with first_window + n_windows < 2^31 (got %lld, %d)",
                static_cast<long long>(first_sample), first_window);
  if (n_windows > 0 && static_cast<int64_t>(static_cast<double>(first_window) * step) < first_sample)
    return fail(LSPG_EINVAL, "window %d starts at sample %lld, before the first sample given (%lld)", first_window,
                static_cast<long long>(static_cast<double>(first_window) * step), static_cast<long long>(first_sample));
  if (int rc = capi::require_device<Lspa>(h->device, "lspa_logmel_at")) return rc;
  if (h->n_mels == 0) return fail(LSPG_ESTATE, "lspa_load_mel_basis has not been called");
  if (n_windows == 0) return LSPG_OK;
  DeviceGuard g(h->device);
  const int blocks = n_windows / kWin + (n_windows % kWin != 0);   // w0 = blockIdx.x * kWin < n_windows < 2^31
  lspa_logmel_kernel<<<blocks, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      audio, first_sample, n_samples, first_window, n_windows, frame_len, step, h->d_tw, h->d_hann, h->d_basis, h->n_mels,
      normalize ? 1 : 0, out);
  CUDA_TRY(cudaGetLastError());
  return LSPG_OK;
}

int lspa_load_resample_filter(lspa_handle h, const double* win, const double* delta, int nwin, int num_table,
                              double sample_ratio) {
  if (!h || !win || !delta) return fail(LSPG_EINVAL, "null argument");
  if (nwin < 2) return fail(LSPG_EINVAL, "nwin must be >= 2 (got %d)", nwin);
  if (num_table < 1) return fail(LSPG_EINVAL, "num_table must be >= 1 (got %d)", num_table);
  if (!(sample_ratio > 0.0) || !(sample_ratio < 1.0e6))
    return fail(LSPG_EINVAL, "sample_ratio must be in (0, 1e6) (got %g)", sample_ratio);
  const double scale = sample_ratio < 1.0 ? sample_ratio : 1.0;
  const int index_step = static_cast<int>(scale * num_table);
  if (index_step < 1)
    return fail(LSPG_EINVAL, "int(min(1, sample_ratio) * num_table) must be >= 1 (got %g * %d)", scale, num_table);
  if (int rc = capi::require_device<Lspa>(h->device, "lspa_load_resample_filter")) return rc;
  DeviceGuard g(h->device);
  h->nwin = 0;                                 // not usable until the copy is complete
  if (h->d_rs_tab) cudaFree(h->d_rs_tab);
  h->d_rs_tab = nullptr;
  double2* tab = new double2[nwin];
  for (int j = 0; j < nwin; ++j) tab[j] = make_double2(win[j], delta[j]);
  cudaError_t e = cudaMalloc(&h->d_rs_tab, sizeof(double2) * nwin);
  if (e == cudaSuccess) e = cudaMemcpy(h->d_rs_tab, tab, sizeof(double2) * nwin, cudaMemcpyHostToDevice);
  delete[] tab;
  if (e != cudaSuccess) return fail(LSPG_ECUDA, "lspa_load_resample_filter: %s", cudaGetErrorString(e));
  h->num_table = num_table;
  h->index_step = index_step;
  h->scale = scale;
  h->nwin = nwin;
  return LSPG_OK;
}

int lspa_resample_at(lspa_handle h, const void* frames, int format, int channels, int64_t first_in, int64_t n_in,
                     int64_t first_out, int64_t n_out, const int64_t* reg_table, int n_reg, float* out, void* stream) {
  if (!h) return fail(LSPG_EINVAL, "null handle");
  if (format != LSPA_FMT_F32 && format != LSPA_FMT_S16) return fail(LSPG_EINVAL, "unknown sample format %d", format);
  if (channels != 1 && channels != 2) return fail(LSPG_EINVAL, "channels must be 1 or 2 (got %d)", channels);
  if (n_in < 0 || n_out < 0 || first_in < 0 || first_out < 0)
    return fail(LSPG_EINVAL, "first_in, n_in, first_out and n_out must be >= 0 (got %lld, %lld, %lld, %lld)",
                static_cast<long long>(first_in), static_cast<long long>(n_in), static_cast<long long>(first_out),
                static_cast<long long>(n_out));
  if (n_in > (INT64_MAX >> 2) || n_out > (INT64_MAX >> 2) || first_out > (INT64_MAX >> 2))
    return fail(LSPG_EINVAL, "counts must be below 2^61");
  if ((!frames && n_in > 0) || (!out && n_out > 0) || !reg_table) return fail(LSPG_EINVAL, "null buffer");
  if (n_reg < 2) return fail(LSPG_EINVAL, "the register table needs a row and the end row (got %d rows)", n_reg);
  const int64_t(*reg)[4] = reinterpret_cast<const int64_t(*)[4]>(reg_table);
  if (reg[0][0] != 0) return fail(LSPG_EINVAL, "the register table must start at output 0");
  for (int i = 0; i + 1 < n_reg; ++i) {
    if (reg[i + 1][0] <= reg[i][0]) return fail(LSPG_EINVAL, "register rows must start at increasing outputs (row %d)", i + 1);
    if (reg[i][1] < 0 || reg[i][2] < 0 || reg[i][3] < -1022 || reg[i][3] > 1023 ||
        reg[i][1] + (reg[i + 1][0] - 1 - reg[i][0]) * static_cast<double>(reg[i][2]) >= 9007199254740992.0)
      return fail(LSPG_EINVAL, "register row %d is out of range", i);
  }
  if (first_out + n_out > reg[n_reg - 1][0])
    return fail(LSPG_EINVAL, "outputs up to %lld requested, the register table ends at %lld",
                static_cast<long long>(first_out + n_out), static_cast<long long>(reg[n_reg - 1][0]));
  if (int rc = capi::require_device<Lspa>(h->device, "lspa_resample_at")) return rc;
  if (h->nwin == 0) return fail(LSPG_ESTATE, "lspa_load_resample_filter has not been called");
  if (n_out == 0) return LSPG_OK;
  int r = 0;
  while (r + 2 < n_reg && reg[r + 1][0] <= first_out) ++r;
  if (first_in > 0) {                          // the left wing of output first_out reads back to n - (nwin / step - 1)
    const int64_t n0 = static_cast<int64_t>(std::ldexp(static_cast<double>(reg[r][1] + (first_out - reg[r][0]) * reg[r][2]),
                                                       static_cast<int>(reg[r][3])));
    if (n0 - (h->nwin / h->index_step - 1) < first_in)
      return fail(LSPG_EINVAL, "output %lld reads input frames from %lld, before the first frame given (%lld)",
                  static_cast<long long>(first_out), static_cast<long long>(n0 - (h->nwin / h->index_step - 1)),
                  static_cast<long long>(first_in));
  }
  DeviceGuard g(h->device);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  for (int64_t t = first_out, end = first_out + n_out; t < end;) {       // one launch per kMaxRegRows register rows
    while (r + 2 < n_reg && reg[r + 1][0] <= t) ++r;
    RegRows rows;
    rows.n = 0;
    for (int i = r; i < n_reg - 1 && rows.n < kMaxRegRows; ++i, ++rows.n) {
      rows.t0[rows.n] = reg[i][0];
      rows.base[rows.n] = reg[i][1];
      rows.k[rows.n] = reg[i][2];
      rows.e[rows.n] = static_cast<int>(reg[i][3]);
    }
    const int64_t stop = std::min(end, reg[r + rows.n][0]);
    const int64_t m = stop - t;
    const int64_t blocks = (m + kRsThreads - 1) / kRsThreads;
    if (blocks > INT32_MAX) return fail(LSPG_EINVAL, "too many outputs in one call (%lld)", static_cast<long long>(m));
    auto kern = format == LSPA_FMT_S16 ? (channels == 1 ? lspa_resample_kernel<LSPA_FMT_S16, 1> : lspa_resample_kernel<LSPA_FMT_S16, 2>)
                                       : (channels == 1 ? lspa_resample_kernel<LSPA_FMT_F32, 1> : lspa_resample_kernel<LSPA_FMT_F32, 2>);
    kern<<<static_cast<unsigned>(blocks), kRsThreads, 0, st>>>(frames, first_in, n_in, t, m, rows, h->d_rs_tab, h->nwin,
                                                                h->num_table, h->index_step, h->scale, out + (t - first_out));
    CUDA_TRY(cudaGetLastError());
    t = stop;
  }
  return LSPG_OK;
}

}  // extern "C"
