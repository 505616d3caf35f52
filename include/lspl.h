/*
 * lspl.h - C ABI of the H100-native landmark post-processing (LiveSpeechPortraits, SURVEY.md 8f row N7).
 *
 * What it replaces: stage 5 of demo.py (:215-255) - in numpy on the host: the mouth track smoothed, amplified, put on
 * the mean face and its crossed inner lips fixed (funcs/utils.py landmark_smooth_3d, mouth_pts_AMP,
 * solve_intersect_mouth), the head pose amplified and smoothed (headpose_smooth), then two Python loops over the frames
 * that project the 73 face landmarks (project_landmarks, angle2matrix) and the 18 shoulder points.  Here two kernels
 * take the device tracks of stages 3 and 4 to the device tracks the rasteriser draws.
 *
 * Conventions as in lspg.h / lspm.h / lspa.h: plain C types, 0 or a negative LSPG_E* code, message in
 * lspl_last_error(); sm_90 only, no CPU path.  lspl_run is asynchronous on `stream`, allocates nothing and does not
 * synchronise the host; its buffers are DEVICE pointers.  The Python binding is livespeechportraits_b200/landmarks.py.
 */
#ifndef LSPL_H_
#define LSPL_H_

#include <stddef.h>
#include <stdint.h>

#include "lspg.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct lspl_ctx* lspl_handle;

/* The identity constants demo.py loads once (:81-108), host arrays in float64 (fp32 files are passed as their exact
 * float64 values).  Rows of the 73-point face are [73][3], row-major. */
typedef struct {
  const double* mean_pts3d;          /* [73][3] mean_pts3d.npy */
  const double* std_mean_pts3d;      /* [73][3] the mean of the identity's pts3d */
  const double* candidate_eye_brow;  /* [m][16][3] pts3d[10:, eye_brow_indices] - mean_pts3d */
  int n_candidates;                  /* m >= 1 */
  double mean_translation[3];        /* fp32 in the reference: rounded to fp32 on load */
  double ref_trans[3];               /* fp32 in the reference: rounded to fp32 on load */
  const double* shoulder3D;          /* [18][3] */
  double camera_intrinsic[9];        /* [3][3], fp32 in the reference: rounded to fp32 on load */
  double relative_rotation[9];       /* camera().relative_rotation, fp32 in the reference: rounded on load */
  double relative_translation[3];    /* camera().relative_translation, fp32 in the reference: rounded on load */
  double scale;                      /* id_scale.mat */
} lspl_identity;

/* The per-clip parameters of config/<id>.yaml. */
typedef struct {
  double feat_sigma;                 /* Audio2Mouth smooth: >= 0, 0 skips the smoothing */
  double rot_sigma, trans_sigma;     /* Headpose smooth: > 0 */
  double amp[18][3];                 /* mouth AMP as one scale per (mouth row 46 + i, coordinate) */
  double rot_amp, trans_amp;         /* Headpose AMP */
  double shoulder_amp;               /* rounded to fp32, as numpy multiplies an fp32 array by a Python float */
  int use_pad;                       /* nonzero: add image_pad to the shoulders after projecting them */
  int pad[4];                        /* top, bottom, left, right: x += right - left, y += top - bottom */
} lspl_params;

/* Smoothing radius int(4 sigma + 0.5) is limited to this; larger sigmas are refused with LSPG_EINVAL. */
#define LSPL_MAX_RADIUS 1024

/* device == -1: host-only handle (argument checking only; lspl_load_identity / lspl_run return LSPG_ENODEV). */
int lspl_create(lspl_handle* out, int device);

/* Synchronous: rounds to fp32 what the reference keeps in fp32, forms the fp32 eyebrow table
 * candidate_eye_brow + mean_pts3d[eye_brow_indices], and copies it all to library-owned device memory.  A second call
 * replaces the identity. */
int lspl_load_identity(lspl_handle h, const lspl_identity* id);

/* Bytes of caller-owned device workspace lspl_run needs for these track lengths. */
int lspl_workspace_bytes(lspl_handle h, int n_feat, int n_head, size_t* out);

/* demo.py :217-255 for nframe = min(n_feat, n_head) frames.
 *   pred_feat [n_feat][75] fp32: the Audio2Feature track, 25 points at mouth_indices (4..10, 46..63).
 *   pred_head [n_head][head_stride] fp32, head_stride >= 6: rotation (degrees) in 0:3, translation in 3:6.
 *   landmarks [nframe][73][2], shoulders [nframe][18][2] fp32 pixel coordinates (pred_landmarks / pred_shoulders; the
 *   shoulders with image_pad added when p->use_pad).  final_pts3d [nframe][73][3] and pred_headpose [nframe][6] fp32
 *   are optional (NULL skips them).  The mouth is smoothed over nframe rows, the head pose over all n_head rows.
 *   nframe == 0 launches nothing.  Identical inputs give bit-identical outputs. */
int lspl_run(lspl_handle h, const float* pred_feat, int n_feat, const float* pred_head, int n_head, int head_stride,
             const lspl_params* p, float* landmarks, float* shoulders, float* final_pts3d, float* pred_headpose,
             void* workspace, size_t workspace_bytes, void* stream);

/* Streaming: the same frames from track rows that arrive in pieces (the live path of livespeechportraits_b200/stream.py).
 *
 * Frame t of a call equals frame t of lspl_run on the whole tracks, value for value, except the outer lips of crossed
 * frames (below).  Row i of the mouth track is feat[i - feat_row0] (n_feat_rows rows given), row i of the head track
 * head[(i - head_row0) * head_stride]; frames frame0 .. frame0 + n_frames - 1 are written to row 0 .. n_frames - 1 of
 * the outputs.  The mouth reflects at nframe_total (= min(n_feat, n_head) of the whole clip), the head at
 * n_head_total, as in lspl_run; each total is -1 while the clip goes on.  The eyebrow candidate is t % m with the
 * global t.
 *
 * Refused with LSPG_EINVAL: a frame at or past a known total; while nframe_total is -1, a frame t with
 * t + rm >= head_row0 + n_head_rows (the mouth window must be interior: nframe may yet end at the head rows); a row
 * window not covered, i.e. the mouth rows max(0, t - rm) .. t + rm and the head rows max(0, t - rh) .. t + rh
 * (rh = max(rr, rt); capped at a known total minus one) must lie in the rows given for every frame emitted.  Rows
 * and frames end at or below 2^29.
 *
 * The live lip fix.  A frame is crossed when all three lower inner-lip y exceed the upper ones (as in lspl_run); its
 * inner lips move by its own half-differences (as in lspl_run).  Its outer lips move by the running mean of
 * half_inner_y_diff over the crossed frames up to and including it: S += h_t, C += 1, shift_t = S / (3 C), with h_t
 * the three-term fp64 sum lspl_run adds up, taken one frame at a time in frame order.  The result does not depend on
 * how the clip was cut into calls; at the last crossed frame the shift equals lspl_run's clip mean up to fp64
 * summation order.  `state` (lspl_stream_state_bytes, device memory) carries S and C between calls; frame0 == 0 starts
 * them from zero.
 *
 * At most three launches on `stream`; allocates nothing, does not synchronise the host, no atomics: identical inputs
 * give bit-identical outputs.  Host-only handles check the arguments and return LSPG_ENODEV. */
int lspl_stream_state_bytes(lspl_handle h, size_t* out);
int lspl_stream_workspace_bytes(lspl_handle h, int n_frames, size_t* out);
int lspl_run_stream(lspl_handle h, const float* feat, int feat_row0, int n_feat_rows, const float* head, int head_row0,
                    int n_head_rows, int head_stride, int frame0, int n_frames, int nframe_total, int n_head_total,
                    const lspl_params* p, float* landmarks, float* shoulders, float* final_pts3d, float* pred_headpose,
                    void* state, void* workspace, size_t workspace_bytes, void* stream);

int lspl_destroy(lspl_handle h);
const char* lspl_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* LSPL_H_ */
