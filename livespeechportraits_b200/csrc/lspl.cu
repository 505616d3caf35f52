// C-ABI implementation of the landmark post-processing (see include/lspl.h; SURVEY.md 8f row N7).
//
// Reference: demo.py :217-255 with funcs/utils.py angle2matrix, project_landmarks, landmark_smooth_3d, mouth_pts_AMP,
// solve_intersect_mouth and headpose_smooth (:182-367).  Two launches, both on the caller's stream:
//   1. lspl_smooth_kernel: one CTA per 32 frames.  Each CTA first builds the normalised gaussian taps of the three
//      sigmas in shared memory (exp(-x^2 / 2 sigma^2) over |x| <= int(4 sigma + 0.5), normalised in fp64, as
//      scipy.ndimage.gaussian_filter1d does).  A thread then owns one (frame, column) of the 54 mouth columns (rows
//      46..63 of pts3d, the only mouth rows that reach the output) or the 6 pose columns, and sums the taps in fp64 in
//      scipy's symmetric order (centre tap, then the pairs from the outermost in), reading the track through the
//      read-only cache with mode='reflect' (period 2N, so clips shorter than the radius fold back more than once).  The
//      mouth is read over nframe rows, the pose over all n_head rows.  Epilogue: the mouth gets its AMP scale and the mean
//      face in fp64; the pose is rounded to fp32, then mean_translation and 180 degrees are added in fp32.  Each CTA
//      decides, per frame, whether all three inner-lip pairs cross, and writes its fp64 sum of the half-differences of
//      those frames and their count.
//   2. lspl_project_kernel: one CTA per 32 frames.  Every CTA sums all the partials of kernel 1 in one fixed order (no
//      atomics), so the clip-wide lip-fix mean is the same everywhere.  One thread per frame then fixes the lips, builds R
//      in fp64 from the fp32 angles (deg2rad in fp32 as numpy evaluates it on an fp32 scalar, math.cos / math.sin in fp64)
//      and rounds it to fp32 as angle2matrix does.  One thread per (frame, point) assembles final_pts3d in fp32 and
//      projects it: the 73 face points in fp64 from those fp32 values, the 18 shoulder points in fp32 as the reference
//      computes them, with image_pad added last.
// lspl_run_stream emits a span of frames from the track rows given (Span: global frame and row indices, reflection at
// the totals once known) through the same two kernels and the same __device__ functions, with a third launch between
// them: lspl_lipfix_scan_kernel replaces the clip-wide lip-fix mean by the running mean over the crossed frames so far.
// Fixed summation orders everywhere: results are bit-identical from run to run.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>

#include "../../include/lspl.h"
#include "capi.cuh"

using capi::DeviceGuard;

namespace {

struct Lspl;
constexpr auto fail = capi::fail<Lspl>;

constexpr int kPts = 73;
constexpr int kMouth0 = 46;                    // rows 46..63 of the face come from the mouth track
constexpr int kMouthCols = 18 * 3;
constexpr int kFeatCols = 75;                  // 25 points at mouth_indices 4..10, 46..63
constexpr int kFeatMouthOff = 7 * 3;           // row 46 is the 8th point of pred_Feat
constexpr int kShoulders = 18;
constexpr int kItems = kPts + kShoulders;      // points projected per frame
constexpr int kFrames = 32;                    // frames per CTA, both kernels
constexpr int kThreads = 256;
constexpr int kMaxN = 1 << 29;                 // t + radius and 2 n stay within int
constexpr unsigned kFull = 0xffffffffu;

struct DevIdentity {
  double mouth_mean[kMouthCols];               // mean_pts3d rows 46..63
  double shoulder3D[kShoulders * 3];
  double scale;
  float std_mean[kPts * 3];                    // std_mean_pts3d rounded to fp32 (final_pts3d is fp32)
  float mean_translation[3], ref_trans[3];
  float K[9], Rv[9], tv[3];
  signed char brow_slot[kPts];                 // slot of the row in eye_brow_indices (demo.py:75), -1 elsewhere
};

struct KParams {
  double amp[kMouthCols];
  double rot_amp, trans_amp;
  int rm, rr, rt;                              // radii; rm == 0 leaves the mouth unsmoothed
  float shoulder_amp, pad_x, pad_y;
  int use_pad;
  float deg2rad;                               // fp32(fp32(pi) / 180), numpy's constant for fp32 deg2rad
};

// The frames one launch emits and the rows it reads.  Frame t (global) is local frame t - frame0 of the outputs and the
// workspace; row i of a track is at (i - row0) of its pointer.  The mouth reflects at n_mouth (nframe of the whole clip),
// the head at n_head; kOpen while the clip goes on (the caller guarantees that no window reaches that far).  lspl_run is
// the span {0, nframe, 0, 0, nframe, n_head}.
struct Span {
  int frame0, n;
  int feat_row0, head_row0;
  int n_mouth, n_head;
};
constexpr int kOpen = (1 << 30) - 1;           // reflect() at kOpen only folds negative indices; 2 kOpen fits an int

struct Workspace {
  double* mouth;                               // [n][54] mouth rows after AMP and the mean face
  float* pose;                                 // [n][6]  pred_headpose
  double* part_sum;                            // whole clip: [ctas] sum of the half-differences of the fixed frames
  int* part_cnt;                               // whole clip: [ctas] number of fixed frames
  double* shift;                               // stream: [n] the outer-lip shift of each frame (running mean)
};

// lspl_run_stream's state: the running sum of half_inner_y_diff over the crossed frames so far, and their count
struct LipState {
  double sum;
  long long count;
};

size_t align_up(size_t x) { return (x + 255) & ~size_t(255); }

Workspace carve(void* base, int n, bool stream, size_t* total) {
  const int ctas = (n + kFrames - 1) / kFrames;
  size_t off = 0;
  Workspace w{};
  char* b = static_cast<char*>(base);
  w.mouth = reinterpret_cast<double*>(b + off);   off = align_up(off + sizeof(double) * kMouthCols * size_t(n));
  w.pose = reinterpret_cast<float*>(b + off);     off = align_up(off + sizeof(float) * 6 * size_t(n));
  if (stream) {
    w.shift = reinterpret_cast<double*>(b + off); off = align_up(off + sizeof(double) * size_t(n));
  } else {
    w.part_sum = reinterpret_cast<double*>(b + off); off = align_up(off + sizeof(double) * size_t(ctas));
    w.part_cnt = reinterpret_cast<int*>(b + off);   off = align_up(off + sizeof(int) * size_t(ctas));
  }
  *total = off;
  return w;
}

int radius_of(double sigma) { return static_cast<int>(4.0 * sigma + 0.5); }

// scipy.ndimage mode='reflect' (d c b a | a b c d | d c b a): period 2n
__device__ __forceinline__ int reflect(int i, int n) {
  if (i >= 0 && i < n) return i;
  const int p = 2 * n;
  int m = i % p;
  if (m < 0) m += p;
  return m < n ? m : p - 1 - m;
}

// where track row i, reflected at n, sits in a buffer whose first row is row0
__device__ __forceinline__ int64_t row_offset(int i, int n, int row0, int stride) {
  return static_cast<int64_t>(reflect(i, n) - row0) * stride;
}

// warp-wide: w[k] = exp(-0.5 / sigma^2 * k^2) / sum_{|x| <= r} exp(...), k = 0..r, fixed lane order then xor tree
__device__ void gaussian_taps(double* w, int r, double sigma, int lane) {
  const double c = -0.5 / (sigma * sigma);
  double s = 0.0;
  for (int k = lane; k <= r; k += 32) {
    const double phi = exp(c * static_cast<double>(k * k));
    w[k] = phi;
    if (k) s += phi;
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) s += __shfl_xor_sync(kFull, s, off);
  const double total = 1.0 + 2.0 * s;
  __syncwarp();
  for (int k = lane; k <= r; k += 32) w[k] /= total;
}

// Mouth column c (of rows 46..63) at frame t: the fp64 gaussian sum in scipy's order (centre tap, then the pairs from
// the outermost in) over the reflected rows, then AMP and the mean face.
__device__ __forceinline__ double mouth_value(const float* __restrict__ feat, const Span& sp, int t, int c,
                                              const double* wm, const KParams& kp, const DevIdentity* __restrict__ id) {
  const float* x = feat + kFeatMouthOff + c;
  const auto row = [&](int i) { return row_offset(i, sp.n_mouth, sp.feat_row0, kFeatCols); };
  double v;
  if (kp.rm == 0) {
    v = static_cast<double>(__ldg(x + row(t)));
  } else {
    v = static_cast<double>(__ldg(x + row(t))) * wm[0];
    for (int k = kp.rm; k >= 1; --k) {
      const double a = __ldg(x + row(t - k));
      const double b = __ldg(x + row(t + k));
      v += (a + b) * wm[k];
    }
  }
  return v * kp.amp[c] + id->mouth_mean[c];
}

// Pose column j at frame t: the fp64 gaussian sum of h * AMP, rounded to fp32, then mean_translation (3..5) or 180 (0)
// added in fp32.
__device__ __forceinline__ float pose_value(const float* __restrict__ head, int head_stride, const Span& sp, int t, int j,
                                            const double* w, int r, const KParams& kp, const DevIdentity* __restrict__ id) {
  const double amp = j < 3 ? kp.rot_amp : kp.trans_amp;
  const float* x = head + j;
  const auto row = [&](int i) { return row_offset(i, sp.n_head, sp.head_row0, head_stride); };
  double v = (static_cast<double>(__ldg(x + row(t))) * amp) * w[0];
  for (int k = r; k >= 1; --k) {
    const double a = static_cast<double>(__ldg(x + row(t - k))) * amp;
    const double b = static_cast<double>(__ldg(x + row(t + k))) * amp;
    v += (a + b) * w[k];
  }
  float pv = static_cast<float>(v);
  if (j >= 3) pv = __fadd_rn(pv, id->mean_translation[j - 3]);
  if (j == 0) pv = __fadd_rn(pv, 180.f);
  return pv;
}

// solve_intersect_mouth on one frame's inner-lip y (upper 63, 62, 61, then lower 58, 59, 60): whether all three pairs
// cross, and half_inner_y_diff summed over the three pairs
__device__ __forceinline__ bool lips_cross(const double* y) { return y[3] > y[0] && y[4] > y[1] && y[5] > y[2]; }
__device__ __forceinline__ double half_diff_sum(const double* y) {
  return (y[3] - y[0]) * 0.5 + (y[4] - y[1]) * 0.5 + (y[5] - y[2]) * 0.5;
}

__global__ void __launch_bounds__(kThreads, 1) lspl_smooth_kernel(const float* __restrict__ feat, const float* __restrict__ head,
                                                                Span sp, int head_stride, double feat_sigma,
                                                                double rot_sigma, double trans_sigma, KParams kp,
                                                                const DevIdentity* __restrict__ id, Workspace ws,
                                                                float* __restrict__ out_pose) {
  extern __shared__ double sw[];               // taps: mouth [rm + 1], rot [rr + 1], trans [rt + 1]
  __shared__ double lip[kFrames][6];           // y of the inner lips: upper 63, 62, 61, then lower 58, 59, 60
  double* wm = sw;
  double* wr = wm + kp.rm + 1;
  double* wt = wr + kp.rr + 1;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (warp == 0 && kp.rm > 0) gaussian_taps(wm, kp.rm, feat_sigma, lane);
  if (warp == 1) gaussian_taps(wr, kp.rr, rot_sigma, lane);
  if (warp == 2) gaussian_taps(wt, kp.rt, trans_sigma, lane);
  __syncthreads();

  const int l0 = blockIdx.x * kFrames;         // local frame of this CTA's first frame
  const int c = tid & 63;
  for (int f = tid >> 6; f < kFrames; f += kThreads / 64) {
    const int l = l0 + f;
    if (l >= sp.n || c >= kMouthCols + 6) continue;
    const int t = sp.frame0 + l;
    if (c < kMouthCols) {
      const double v = mouth_value(feat, sp, t, c, wm, kp, id);
      ws.mouth[static_cast<int64_t>(l) * kMouthCols + c] = v;
      const int row = kMouth0 + c / 3;
      if (c % 3 == 1 && row >= 58 && row <= 63) lip[f][row >= 61 ? 63 - row : 3 + row - 58] = v;
    } else {
      const int j = c - kMouthCols;
      const float pv = pose_value(head, head_stride, sp, t, j, j < 3 ? wr : wt, j < 3 ? kp.rr : kp.rt, kp, id);
      ws.pose[static_cast<int64_t>(l) * 6 + j] = pv;
      if (out_pose) out_pose[static_cast<int64_t>(l) * 6 + j] = pv;
    }
  }
  if (!ws.part_sum) return;                    // a stream: lspl_lipfix_scan_kernel takes the running mean instead
  __syncthreads();

  // solve_intersect_mouth, the clip-wide part: frames whose three lower inner y all exceed the upper ones
  if (warp == 0) {
    const int l = l0 + lane;
    double s = 0.0;
    int cnt = 0;
    if (l < sp.n && lips_cross(lip[lane])) {
      s = half_diff_sum(lip[lane]);
      cnt = 1;
    }
#pragma unroll
    for (int off = 16; off; off >>= 1) {
      s += __shfl_xor_sync(kFull, s, off);
      cnt += __shfl_xor_sync(kFull, cnt, off);
    }
    if (lane == 0) {
      ws.part_sum[blockIdx.x] = s;
      ws.part_cnt[blockIdx.x] = cnt;
    }
  }
}

// The live lip fix (streams only): one warp walks the call's frames in order.  Each lane tests one frame of a group of
// 32; lane 0 then adds the crossed frames' half_diff_sum to the running sum one at a time, so the result does not
// depend on how the clip was cut into calls, and stores each frame's S / (3 C).
__global__ void __launch_bounds__(32) lspl_lipfix_scan_kernel(int n, int reset, Workspace ws, LipState* __restrict__ state) {
  __shared__ double h[32];
  __shared__ int fl[32];
  const int lane = threadIdx.x;
  double s = 0.0;
  long long cnt = 0;
  if (lane == 0 && !reset) {
    s = state->sum;
    cnt = state->count;
  }
  for (int l0 = 0; l0 < n; l0 += 32) {
    const int l = l0 + lane;
    if (l < n) {
      const double* m = ws.mouth + static_cast<int64_t>(l) * kMouthCols;
      const double y[6] = {m[(63 - kMouth0) * 3 + 1], m[(62 - kMouth0) * 3 + 1], m[(61 - kMouth0) * 3 + 1],
                           m[(58 - kMouth0) * 3 + 1], m[(59 - kMouth0) * 3 + 1], m[(60 - kMouth0) * 3 + 1]};
      fl[lane] = lips_cross(y);
      h[lane] = fl[lane] ? half_diff_sum(y) : 0.0;
    }
    __syncwarp();
    if (lane == 0) {
      const int k = min(32, n - l0);
      for (int i = 0; i < k; ++i) {
        if (fl[i]) {
          s += h[i];
          ++cnt;
        }
        ws.shift[l0 + i] = cnt ? s / (3.0 * static_cast<double>(cnt)) : 0.0;
      }
    }
    __syncwarp();
  }
  if (lane == 0) {
    state->sum = s;
    state->count = cnt;
  }
}

// angle2matrix: R = Rz Ry Rx in fp64 from the fp32 angles (deg2rad in fp32), rounded to fp32
__device__ __forceinline__ void rotation(const float* pose, const KParams& kp, float* R) {
  double cs[3], sn[3];
  for (int k = 0; k < 3; ++k) {
    const double a = static_cast<double>(__fmul_rn(pose[k], kp.deg2rad));
    cs[k] = cos(a);
    sn[k] = sin(a);
  }
  const double Rx[3][3] = {{1, 0, 0}, {0, cs[0], -sn[0]}, {0, sn[0], cs[0]}};
  const double Ry[3][3] = {{cs[1], 0, sn[1]}, {0, 1, 0}, {-sn[1], 0, cs[1]}};
  const double Rz[3][3] = {{cs[2], -sn[2], 0}, {sn[2], cs[2], 0}, {0, 0, 1}};
  double M[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) M[i][j] = Ry[i][0] * Rx[0][j] + Ry[i][1] * Rx[1][j] + Ry[i][2] * Rx[2][j];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) R[i * 3 + j] = static_cast<float>(Rz[i][0] * M[0][j] + Rz[i][1] * M[1][j] + Rz[i][2] * M[2][j]);
}

// project_landmarks for one face point: scale * R p + trans, viewpoint, intrinsics, z divide; fp64 from the fp32 values
__device__ __forceinline__ float2 project_face(const float* p, const float* R, const float* T, const DevIdentity* __restrict__ id) {
  double X[3], V[3], P[3];
  for (int i = 0; i < 3; ++i) {
    const double rp = static_cast<double>(R[i * 3]) * p[0] + static_cast<double>(R[i * 3 + 1]) * p[1] +
                      static_cast<double>(R[i * 3 + 2]) * p[2];
    X[i] = id->scale * rp + static_cast<double>(T[i]);
  }
  for (int i = 0; i < 3; ++i)
    V[i] = static_cast<double>(id->Rv[i * 3]) * X[0] + static_cast<double>(id->Rv[i * 3 + 1]) * X[1] +
           static_cast<double>(id->Rv[i * 3 + 2]) * X[2] + static_cast<double>(id->tv[i]);
  for (int i = 0; i < 3; ++i)
    P[i] = static_cast<double>(id->K[i * 3]) * V[0] + static_cast<double>(id->K[i * 3 + 1]) * V[1] +
           static_cast<double>(id->K[i * 3 + 2]) * V[2];
  return make_float2(static_cast<float>(P[0] / P[2]), static_cast<float>(P[1] / P[2]));
}

// shoulder point s: shoulder3D + (pose[3:] - ref_trans) * shoulder_AMP, through the intrinsics, in fp32, plus image_pad
__device__ __forceinline__ float2 project_shoulder(int s, const float* T, const KParams& kp, const DevIdentity* __restrict__ id) {
  float x[3];
  for (int i = 0; i < 3; ++i) {
    const float d = __fmul_rn(__fsub_rn(T[i], id->ref_trans[i]), kp.shoulder_amp);
    x[i] = static_cast<float>(id->shoulder3D[s * 3 + i] + static_cast<double>(d));
  }
  float P[3];
  for (int i = 0; i < 3; ++i)
    P[i] = __fadd_rn(__fadd_rn(__fmul_rn(id->K[i * 3], x[0]), __fmul_rn(id->K[i * 3 + 1], x[1])),
                     __fmul_rn(id->K[i * 3 + 2], x[2]));
  float u = __fdiv_rn(P[0], P[2]), v = __fdiv_rn(P[1], P[2]);
  if (kp.use_pad) { u = __fadd_rn(u, kp.pad_x); v = __fadd_rn(v, kp.pad_y); }
  return make_float2(u, v);
}

// n_parts > 0 (whole clip): the outer lips move by the mean over all crossed frames of the clip, from the partials of
// lspl_smooth_kernel.  n_parts == 0 (stream): by ws.shift of their own frame.
__global__ void __launch_bounds__(kThreads) lspl_project_kernel(Span sp, int n_parts, KParams kp,
                                                                 const DevIdentity* __restrict__ id,
                                                                 const float* __restrict__ brow, int n_brow, Workspace ws,
                                                                 float* __restrict__ landmarks, float* __restrict__ shoulders,
                                                                 float* __restrict__ final_pts3d) {
  __shared__ double red[kThreads];
  __shared__ int redc[kThreads];
  __shared__ float R[kFrames][9];
  __shared__ float T[kFrames][3];
  __shared__ double half[kFrames][3];
  __shared__ double outer[kFrames];
  __shared__ int flip[kFrames];
  __shared__ double outer_shift;
  const int tid = threadIdx.x;
  const int l0 = blockIdx.x * kFrames;

  // the mean of half_inner_y_diff over all fixed frames x 3: same order in every CTA
  if (n_parts) {
    double s = 0.0;
    int cnt = 0;
    for (int i = tid; i < n_parts; i += kThreads) { s += ws.part_sum[i]; cnt += ws.part_cnt[i]; }
    red[tid] = s;
    redc[tid] = cnt;
    __syncthreads();
    for (int h = kThreads / 2; h; h >>= 1) {
      if (tid < h) { red[tid] += red[tid + h]; redc[tid] += redc[tid + h]; }
      __syncthreads();
    }
    if (tid == 0) outer_shift = redc[0] ? red[0] / (3.0 * redc[0]) : 0.0;
  }

  if (tid < kFrames && l0 + tid < sp.n) {
    const int64_t l = l0 + tid;
    const double* m = ws.mouth + l * kMouthCols;
    const double y[6] = {m[(63 - kMouth0) * 3 + 1], m[(62 - kMouth0) * 3 + 1], m[(61 - kMouth0) * 3 + 1],
                         m[(58 - kMouth0) * 3 + 1], m[(59 - kMouth0) * 3 + 1], m[(60 - kMouth0) * 3 + 1]};
    const int fl = lips_cross(y);
    flip[tid] = fl;
    for (int j = 0; j < 3; ++j) half[tid][j] = fl ? (y[3 + j] - y[j]) * 0.5 : 0.0;
    if (!n_parts) outer[tid] = ws.shift[l];
    rotation(ws.pose + l * 6, kp, R[tid]);
    for (int k = 0; k < 3; ++k) T[tid][k] = ws.pose[l * 6 + 3 + k];
  }
  __syncthreads();

  const int nf = min(kFrames, sp.n - l0);
  for (int e = tid; e < nf * kItems; e += kThreads) {
    const int f = e / kItems, q = e - f * kItems;
    const int64_t l = l0 + f;
    if (q < kPts) {
      float p[3];
      const int slot = id->brow_slot[q];
      if (slot >= 0) {
        const int64_t t = sp.frame0 + l;                        // the eyebrow candidate follows the global frame
        const float* b = brow + (static_cast<int64_t>(t % n_brow) * 16 + slot) * 3;
        p[0] = b[0]; p[1] = b[1]; p[2] = b[2];
      } else if (q >= kMouth0 && q < kMouth0 + 18) {
        const double* m = ws.mouth + l * kMouthCols + (q - kMouth0) * 3;
        double y = m[1];
        if (flip[f]) {
          const double shift = n_parts ? outer_shift : outer[f];
          if (q >= 61) y += half[f][63 - q];                    // upper inner 63, 62, 61
          else if (q >= 58) y -= half[f][q - 58];               // lower inner 58, 59, 60
          else if (q >= 47 && q <= 51) y += shift;              // upper outer
          else if (q >= 53) y -= shift;                         // lower outer 57..53
        }
        p[0] = static_cast<float>(m[0]); p[1] = static_cast<float>(y); p[2] = static_cast<float>(m[2]);
      } else {
        p[0] = id->std_mean[q * 3]; p[1] = id->std_mean[q * 3 + 1]; p[2] = id->std_mean[q * 3 + 2];
      }
      if (final_pts3d) {
        float* o = final_pts3d + (l * kPts + q) * 3;
        o[0] = p[0]; o[1] = p[1]; o[2] = p[2];
      }
      *reinterpret_cast<float2*>(landmarks + (l * kPts + q) * 2) = project_face(p, R[f], T[f], id);
    } else {
      const int s = q - kPts;
      *reinterpret_cast<float2*>(shoulders + (l * kShoulders + s) * 2) = project_shoulder(s, T[f], kp, id);
    }
  }
}

}  // namespace

struct lspl_ctx {
  int device = -1;
  int n_brow = 0;                              // 0 until an identity is loaded
  DevIdentity* d_id = nullptr;
  float* d_brow = nullptr;                     // [n_brow][16][3]
};

extern "C" {

const char* lspl_last_error(void) { return capi::last_error<Lspl>().c_str(); }

int lspl_destroy(lspl_handle h) {
  if (!h) return LSPG_OK;
  if (h->device >= 0) {
    DeviceGuard g(h->device);
    if (h->d_id) cudaFree(h->d_id);
    if (h->d_brow) cudaFree(h->d_brow);
  }
  delete h;
  return LSPG_OK;
}

int lspl_create(lspl_handle* out, int device) {
  if (!out) return fail(LSPG_EINVAL, "null argument");
  *out = nullptr;
  cudaDeviceProp prop;
  if (int rc = capi::check_device<Lspl>(device, &prop)) return rc;
  lspl_ctx* h = new lspl_ctx;
  h->device = device;
  if (device >= 0) {
    DeviceGuard g(device);
    cudaError_t e = cudaMalloc(&h->d_id, sizeof(DevIdentity));
    if (e != cudaSuccess) {
      lspl_destroy(h);
      return fail(LSPG_ECUDA, "lspl_create: %s", cudaGetErrorString(e));
    }
  }
  *out = h;
  return LSPG_OK;
}

int lspl_load_identity(lspl_handle h, const lspl_identity* id) {
  if (!h || !id) return fail(LSPG_EINVAL, "null argument");
  if (!id->mean_pts3d || !id->std_mean_pts3d || !id->candidate_eye_brow || !id->shoulder3D)
    return fail(LSPG_EINVAL, "null identity array");
  if (id->n_candidates < 1) return fail(LSPG_EINVAL, "n_candidates must be >= 1 (got %d)", id->n_candidates);
  if (int rc = capi::require_device<Lspl>(h->device, "lspl_load_identity")) return rc;
  static const int brow_rows[16] = {27, 65, 28, 68, 29, 67, 30, 66, 31, 72, 32, 69, 33, 70, 34, 71};
  DevIdentity d{};
  for (int i = 0; i < kMouthCols; ++i) d.mouth_mean[i] = id->mean_pts3d[kMouth0 * 3 + i];
  for (int i = 0; i < kShoulders * 3; ++i) d.shoulder3D[i] = id->shoulder3D[i];
  d.scale = id->scale;
  for (int i = 0; i < kPts * 3; ++i) d.std_mean[i] = static_cast<float>(id->std_mean_pts3d[i]);
  for (int i = 0; i < 3; ++i) {
    d.mean_translation[i] = static_cast<float>(id->mean_translation[i]);
    d.ref_trans[i] = static_cast<float>(id->ref_trans[i]);
    d.tv[i] = static_cast<float>(id->relative_translation[i]);
  }
  for (int i = 0; i < 9; ++i) {
    d.K[i] = static_cast<float>(id->camera_intrinsic[i]);
    d.Rv[i] = static_cast<float>(id->relative_rotation[i]);
  }
  for (int q = 0; q < kPts; ++q) d.brow_slot[q] = -1;
  for (int s = 0; s < 16; ++s) d.brow_slot[brow_rows[s]] = static_cast<signed char>(s);
  const int m = id->n_candidates;
  float* brow = new float[static_cast<size_t>(m) * 48];
  for (int k = 0; k < m; ++k)
    for (int s = 0; s < 16; ++s)
      for (int c = 0; c < 3; ++c)
        brow[(k * 16 + s) * 3 + c] = static_cast<float>(id->candidate_eye_brow[(static_cast<size_t>(k) * 16 + s) * 3 + c] +
                                                        id->mean_pts3d[brow_rows[s] * 3 + c]);
  DeviceGuard g(h->device);
  h->n_brow = 0;                               // not usable until the copies are complete
  cudaError_t e = cudaSuccess;
  if (h->d_brow) e = cudaFree(h->d_brow);
  h->d_brow = nullptr;
  if (e == cudaSuccess) e = cudaMalloc(&h->d_brow, sizeof(float) * 48 * static_cast<size_t>(m));
  if (e == cudaSuccess) e = cudaMemcpy(h->d_brow, brow, sizeof(float) * 48 * static_cast<size_t>(m), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(h->d_id, &d, sizeof(d), cudaMemcpyHostToDevice);
  delete[] brow;
  if (e != cudaSuccess) return fail(LSPG_ECUDA, "lspl_load_identity: %s", cudaGetErrorString(e));
  h->n_brow = m;
  return LSPG_OK;
}

int lspl_workspace_bytes(lspl_handle h, int n_feat, int n_head, size_t* out) {
  if (!h || !out) return fail(LSPG_EINVAL, "null argument");
  if (n_feat < 0 || n_head < 0 || n_feat > kMaxN || n_head > kMaxN)
    return fail(LSPG_EINVAL, "track lengths must be in [0, 2^29] (got %d, %d)", n_feat, n_head);
  carve(nullptr, n_feat < n_head ? n_feat : n_head, false, out);
  return LSPG_OK;
}

int lspl_stream_state_bytes(lspl_handle h, size_t* out) {
  if (!h || !out) return fail(LSPG_EINVAL, "null argument");
  *out = sizeof(LipState);
  return LSPG_OK;
}

int lspl_stream_workspace_bytes(lspl_handle h, int n_frames, size_t* out) {
  if (!h || !out) return fail(LSPG_EINVAL, "null argument");
  if (n_frames < 0 || n_frames > kMaxN) return fail(LSPG_EINVAL, "n_frames must be in [0, 2^29] (got %d)", n_frames);
  carve(nullptr, n_frames, true, out);
  return LSPG_OK;
}

}  // extern "C"

namespace {

// The checks lspl_run and lspl_run_stream share: sigmas, stride, output pointers; fills the kernels' parameters.
int check_params(const lspl_params* p, int head_stride, const float* landmarks, const float* shoulders, int n, KParams* kp) {
  if (head_stride < 6) return fail(LSPG_EINVAL, "head_stride must be >= 6 (got %d)", head_stride);
  if (!(p->feat_sigma >= 0.0) || radius_of(p->feat_sigma) > LSPL_MAX_RADIUS)
    return fail(LSPG_EINVAL, "feat_sigma must be >= 0 with int(4 sigma + 0.5) <= %d (got %g)", LSPL_MAX_RADIUS, p->feat_sigma);
  if (!(p->rot_sigma > 0.0) || !(p->trans_sigma > 0.0) || radius_of(p->rot_sigma) > LSPL_MAX_RADIUS ||
      radius_of(p->trans_sigma) > LSPL_MAX_RADIUS)
    return fail(LSPG_EINVAL, "head sigmas must be > 0 with int(4 sigma + 0.5) <= %d (got %g, %g): scipy's "
                 "gaussian_filter1d divides by zero at 0", LSPL_MAX_RADIUS, p->rot_sigma, p->trans_sigma);
  if (n > 0 && (!landmarks || !shoulders)) return fail(LSPG_EINVAL, "null output buffer");
  if (reinterpret_cast<uintptr_t>(landmarks) % 8 || reinterpret_cast<uintptr_t>(shoulders) % 8)
    return fail(LSPG_EINVAL, "landmarks and shoulders must be 8-byte aligned");
  *kp = KParams{};
  for (int i = 0; i < kMouthCols; ++i) kp->amp[i] = p->amp[i / 3][i % 3];
  kp->rot_amp = p->rot_amp;
  kp->trans_amp = p->trans_amp;
  kp->rm = p->feat_sigma > 0.0 ? radius_of(p->feat_sigma) : 0;
  kp->rr = radius_of(p->rot_sigma);
  kp->rt = radius_of(p->trans_sigma);
  kp->shoulder_amp = static_cast<float>(p->shoulder_amp);
  kp->use_pad = p->use_pad ? 1 : 0;
  kp->pad_x = static_cast<float>(p->pad[3] - p->pad[2]);
  kp->pad_y = static_cast<float>(p->pad[0] - p->pad[1]);
  kp->deg2rad = 3.14159265358979323846f / 180.0f;
  return LSPG_OK;
}

// lspl_smooth_kernel, then (streams) lspl_lipfix_scan_kernel, then lspl_project_kernel, on `stream`
int launch(lspl_handle h, const float* feat, const float* head, int head_stride, const Span& sp, const lspl_params* p,
           const KParams& kp, float* landmarks, float* shoulders, float* final_pts3d, float* pred_headpose,
           LipState* state, const Workspace& ws, void* stream) {
  DeviceGuard g(h->device);
  const int ctas = (sp.n + kFrames - 1) / kFrames;
  const size_t smem = sizeof(double) * static_cast<size_t>(kp.rm + kp.rr + kp.rt + 3);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  lspl_smooth_kernel<<<ctas, kThreads, smem, st>>>(feat, head, sp, head_stride, p->feat_sigma, p->rot_sigma,
                                                   p->trans_sigma, kp, h->d_id, ws, pred_headpose);
  CUDA_TRY(cudaGetLastError());
  if (state) {
    lspl_lipfix_scan_kernel<<<1, 32, 0, st>>>(sp.n, sp.frame0 == 0, ws, state);
    CUDA_TRY(cudaGetLastError());
  }
  lspl_project_kernel<<<ctas, kThreads, 0, st>>>(sp, state ? 0 : ctas, kp, h->d_id, h->d_brow, h->n_brow, ws, landmarks,
                                                 shoulders, final_pts3d);
  CUDA_TRY(cudaGetLastError());
  return LSPG_OK;
}

// rows [lo, hi) of a track must lie in the rows [row0, row0 + n) given
int check_rows(const char* what, int64_t lo, int64_t hi, int row0, int n) {
  if (lo < row0 || hi > static_cast<int64_t>(row0) + n)
    return fail(LSPG_EINVAL, "%s rows %lld .. %lld are needed, rows %d .. %lld were given", what, static_cast<long long>(lo),
                static_cast<long long>(hi) - 1, row0, static_cast<long long>(row0) + n - 1);
  return LSPG_OK;
}

}  // namespace

extern "C" {

int lspl_run(lspl_handle h, const float* pred_feat, int n_feat, const float* pred_head, int n_head, int head_stride,
             const lspl_params* p, float* landmarks, float* shoulders, float* final_pts3d, float* pred_headpose,
             void* workspace, size_t workspace_bytes, void* stream) {
  if (!h || !p) return fail(LSPG_EINVAL, "null argument");
  if (n_feat < 0 || n_head < 0 || n_feat > kMaxN || n_head > kMaxN)
    return fail(LSPG_EINVAL, "track lengths must be in [0, 2^29] (got %d, %d)", n_feat, n_head);
  const int nframe = n_feat < n_head ? n_feat : n_head;
  KParams kp;
  if (int rc = check_params(p, head_stride, landmarks, shoulders, 0, &kp)) return rc;
  if ((!pred_feat && n_feat > 0) || (!pred_head && n_head > 0)) return fail(LSPG_EINVAL, "null input track");
  if (nframe > 0 && (!landmarks || !shoulders)) return fail(LSPG_EINVAL, "null output buffer");
  if (int rc = capi::require_device<Lspl>(h->device, "lspl_run")) return rc;
  if (h->n_brow == 0) return fail(LSPG_ESTATE, "lspl_load_identity has not been called");
  if (nframe == 0) return LSPG_OK;
  size_t need = 0;
  carve(nullptr, nframe, false, &need);
  if (!workspace || workspace_bytes < need)
    return fail(LSPG_ESTATE, "workspace of %zu bytes is smaller than the %zu lspl_workspace_bytes gives", workspace_bytes, need);
  const Workspace ws = carve(workspace, nframe, false, &need);
  const Span sp{0, nframe, 0, 0, nframe, n_head};
  return launch(h, pred_feat, pred_head, head_stride, sp, p, kp, landmarks, shoulders, final_pts3d, pred_headpose, nullptr,
                ws, stream);
}

int lspl_run_stream(lspl_handle h, const float* feat, int feat_row0, int n_feat_rows, const float* head, int head_row0,
                    int n_head_rows, int head_stride, int frame0, int n_frames, int nframe_total, int n_head_total,
                    const lspl_params* p, float* landmarks, float* shoulders, float* final_pts3d, float* pred_headpose,
                    void* state, void* workspace, size_t workspace_bytes, void* stream) {
  if (!h || !p) return fail(LSPG_EINVAL, "null argument");
  if (!state) return fail(LSPG_EINVAL, "null state");
  if (feat_row0 < 0 || n_feat_rows < 0 || head_row0 < 0 || n_head_rows < 0 || frame0 < 0 || n_frames < 0 ||
      static_cast<int64_t>(feat_row0) + n_feat_rows > kMaxN || static_cast<int64_t>(head_row0) + n_head_rows > kMaxN ||
      static_cast<int64_t>(frame0) + n_frames > kMaxN)
    return fail(LSPG_EINVAL, "rows and frames must be >= 0 and end at or below 2^29 (got feat %d + %d, head %d + %d, "
                "frames %d + %d)", feat_row0, n_feat_rows, head_row0, n_head_rows, frame0, n_frames);
  if (nframe_total < -1 || nframe_total > kMaxN || n_head_total < -1 || n_head_total > kMaxN)
    return fail(LSPG_EINVAL, "nframe_total and n_head_total must be -1 (clip goes on) or in [0, 2^29] (got %d, %d)",
                nframe_total, n_head_total);
  if (nframe_total >= 0 && n_head_total >= 0 && nframe_total > n_head_total)
    return fail(LSPG_EINVAL, "nframe_total %d exceeds n_head_total %d", nframe_total, n_head_total);
  KParams kp;
  if (int rc = check_params(p, head_stride, landmarks, shoulders, n_frames, &kp)) return rc;
  if ((!feat && n_feat_rows > 0) || (!head && n_head_rows > 0)) return fail(LSPG_EINVAL, "null input track");
  if (n_frames > 0) {
    const int64_t t0 = frame0, t1 = static_cast<int64_t>(frame0) + n_frames - 1;
    if ((nframe_total >= 0 && t1 >= nframe_total) || (n_head_total >= 0 && t1 >= n_head_total))
      return fail(LSPG_EINVAL, "frame %lld is past the end of the clip (nframe_total %d, n_head_total %d)",
                  static_cast<long long>(t1), nframe_total, n_head_total);
    const int rh = kp.rr > kp.rt ? kp.rr : kp.rt;
    const int64_t head_in = static_cast<int64_t>(head_row0) + n_head_rows;
    if (nframe_total < 0 && t1 + kp.rm >= head_in)
      return fail(LSPG_EINVAL, "frame %lld is not interior: its mouth window reaches row %lld, and nframe may end at the "
                  "%lld head rows received", static_cast<long long>(t1), static_cast<long long>(t1 + kp.rm),
                  static_cast<long long>(head_in));
    const int64_t mhi = nframe_total >= 0 ? std::min<int64_t>(nframe_total, t1 + kp.rm + 1) : t1 + kp.rm + 1;
    if (int rc = check_rows("mouth", std::max<int64_t>(0, t0 - kp.rm), mhi, feat_row0, n_feat_rows)) return rc;
    const int64_t hhi = n_head_total >= 0 ? std::min<int64_t>(n_head_total, t1 + rh + 1) : t1 + rh + 1;
    if (int rc = check_rows("head", std::max<int64_t>(0, t0 - rh), hhi, head_row0, n_head_rows)) return rc;
  }
  if (int rc = capi::require_device<Lspl>(h->device, "lspl_run_stream")) return rc;
  if (h->n_brow == 0) return fail(LSPG_ESTATE, "lspl_load_identity has not been called");
  if (n_frames == 0) return LSPG_OK;
  size_t need = 0;
  carve(nullptr, n_frames, true, &need);
  if (!workspace || workspace_bytes < need)
    return fail(LSPG_ESTATE, "workspace of %zu bytes is smaller than the %zu lspl_stream_workspace_bytes gives",
                workspace_bytes, need);
  const Workspace ws = carve(workspace, n_frames, true, &need);
  const Span sp{frame0, n_frames, feat_row0, head_row0, nframe_total >= 0 ? nframe_total : kOpen,
                n_head_total >= 0 ? n_head_total : kOpen};
  return launch(h, feat, head, head_stride, sp, p, kp, landmarks, shoulders, final_pts3d, pred_headpose,
                static_cast<LipState*>(state), ws, stream);
}

}  // extern "C"
