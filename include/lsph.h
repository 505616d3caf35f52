/*
 * lsph.h - C ABI of the H100-native Audio2Headpose generation loop (LiveSpeechPortraits, SURVEY.md 8f row N4).
 *
 * What it replaces: the autoregressive loop of models/audio2headpose_model.py:169-187 - per generated frame one
 * Audio2Headpose.forward (models/audio2headpose.py:41-53: audio_downsample of a 255-row window + a 255-step WaveNet,
 * models/networks.py:199-227 / 303-326), a device->host copy, Sample_GMM on the CPU (models/losses.py:68-112) and a
 * host->device copy of the updated history - by ONE persistent kernel that runs the whole clip on the device:
 * the WaveNet is evaluated incrementally (one new time step per frame against per-layer activation histories, which is
 * the same function because the receptive field equals the window length - see csrc/lsph.cu), the audio path and the
 * conditioning convolutions, which do not depend on the generated history, are hoisted out of the loop as three GEMMs, and
 * Sample_GMM runs on the device with the random draws passed in.
 *
 * Conventions as in lspg.h: plain C types, 0 or a negative LSPG_E* code, message in lsph_last_error(); sm_90 only,
 * no CPU path.  The Python binding (livespeechportraits_b200/headpose.py) keeps the reference's
 * generate_sequences(audio_feats, pre_headpose, fill_zero, sigma_scale, opt) signature.
 */
#ifndef LSPH_H_
#define LSPH_H_

#include <stddef.h>
#include <stdint.h>

#include "lspg.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct lsph_ctx* lsph_handle;

/* The option fields Audio2Headpose.__init__ / WaveNet.__init__ read (options/base_options_audio2headpose.py:38-78). */
typedef struct lsph_config {
  int apc_hidden;       /* APC_hidden_size (512): audio feature rows are 2*apc_hidden wide */
  int frame_future;     /* frame_future (15) */
  int layers, blocks;   /* A2H_wavenet_residual_layers (7), A2H_wavenet_residual_blocks (2) */
  int residual_ch;      /* A2H_wavenet_residual_channels (128) - must be 128 */
  int dilation_ch;      /* A2H_wavenet_dilation_channels (128) - must be 128 */
  int skip_ch;          /* A2H_wavenet_skip_channels (256) - must be 256 */
  int kernel_size;      /* A2H_wavenet_kernel_size (2) - must be 2 */
  int use_bias;         /* A2H_wavenet_use_bias (1) */
  int cond_ch;          /* A2H_wavenet_cond_channels (512) = apc_hidden */
  int input_ch;         /* A2H_wavenet_input_channels (12), <= 32 */
  int ncenter, ndim;    /* A2H_GMM_ncenter (1), A2H_GMM_ndim (12); ndim == input_ch (the sample is fed back) */
  int loss_gmm;         /* 1: opt.loss == 'GMM' (output (2*ndim+1)*ncenter <= 128), 0: 'L2' (output ndim) */
} lsph_config;

/* Replaces Audio2Headpose.__init__ (models/audio2headpose.py:8-37) + init_net's device move.  device == -1: host-only
 * handle (weight packing introspection; lsph_generate_stream returns LSPG_ENODEV). */
int lsph_create(lsph_handle* out, const lsph_config* cfg, int device);

/* Replaces load_state_dict of the Audio2Headpose module (models/base_model.py:193-223): keys as in
 * Audio2Headpose(opt).state_dict() ("audio_downsample.0.weight", "WaveNet.residual_blocks.3.filter_conv.weight", ...),
 * optional "module." prefix, host fp32.  Eval-mode BatchNorm1d is folded into the first linear layer's epilogue.
 * Every parameter must be present (LSPG_ESTATE otherwise: there is no initialiser on this side). */
int lsph_load_weights(lsph_handle h, const lspg_tensor* tensors, int n);

/* Bytes of the state of one stream (works on a host-only handle): fp32 [L][ring][residual_ch] history ring - the input of
 * block l at absolute step t sits in slot t mod ring, ring the smallest power of two above the largest dilation (128 for
 * the shipped options) - then 32 floats holding the network input of the next step (the last sample). */
int lsph_state_bytes(lsph_handle h, size_t* bytes);

/* Bytes of device workspace lsph_generate_stream needs for n_audio audio rows.  After a call the workspace holds, as fp32
 * arrays each padded to a multiple of 64 floats, in this order: ds1 [n_audio][apc_hidden] (audio_downsample's first
 * Linear, BatchNorm and LeakyReLU), ds2 [n_audio][apc_hidden] (its second Linear) and cond
 * [n_audio][layers*blocks][2*residual_ch] (each block's cond filter then cond gate projection plus both biases). */
int lsph_stream_workspace_bytes(lsph_handle h, int n_audio, size_t* bytes);

/* Replaces Audio2HeadposeModel.generate_sequences (models/audio2headpose_model.py:133-187; WaveNet decoder,
 * fill_zero=True) on frames frame0 .. frame0 + n_frames - 1 of the head-pose track.  A clip of n_audio audio rows has
 * n_audio - frame_future frames; the whole clip is one call with frame0 = 0, audio_row0 = 0 and
 * n_frames = n_audio - frame_future, and calls with consecutive frame ranges starting at 0 give, concatenated, the same
 * rows bit for bit: the hoisted GEMMs are computed row by row and the loop runs the same steps in the same order.
 * All pointers are DEVICE pointers, fp32, contiguous:
 *   audio_feats  [n_audio, 2*apc_hidden] (the reshape at :148 already applied): the clip's audio rows audio_row0 ..
 *                audio_row0 + n_audio - 1.  They must cover rows frame0 + frame_future .. frame0 + n_frames - 1 +
 *                frame_future, and from row 0 when frame0 == 0 (the rf - 1 warm-up steps that replay window 0 read rows
 *                0 .. frame_future - 1).  Frame i needs audio up to row i + frame_future and nothing later.
 *   pre_headpose [input_ch]                (demo.py:211: zeros)
 *   noise        [n_frames, ndim]: the torch.randn draws of Sample_GMM (losses.py:96), one row per frame
 *   uniform      [n_frames] or NULL: one U(0,1) draw per frame selecting the mixture component when ncenter > 1 (inverse
 *                CDF of the softmax weights; torch.multinomial's own stream is not reproduced)
 *   out_pred     [n_frames, ndim] = pred_headpose (:186)
 *   out_params   [n_frames, out_ch] or NULL: the network output (GMM parameters) of every frame
 *   state        lsph_state_bytes of caller-owned device memory, 16-byte aligned.  frame0 == 0 starts the loop from
 *                pre_headpose (the ring needs no clearing: reads before step 0 are window 0's zero padding); every call
 *                leaves the state after its last frame, which the call for frame0 + n_frames continues from.
 *   ws           lsph_stream_workspace_bytes(h, n_audio) bytes, 256-byte aligned.
 * cluster: CTAs that share a frame's work (1 or 8; 0 = library default).  n_frames == 0 does nothing.  LSPG_EINVAL
 * (checked before the device, so also on a host-only handle) for a null state or audio rows that do not cover the frames;
 * LSPG_ENODEV on a host-only handle.  Asynchronous on `stream`. */
int lsph_generate_stream(lsph_handle h, const float* audio_feats, int audio_row0, int n_audio, int frame0, int n_frames,
                         const float* pre_headpose, const float* noise, const float* uniform, float sigma_scale,
                         float* out_pred, float* out_params, float* state, void* ws, size_t ws_bytes, int cluster,
                         void* stream);

/* Receptive field of the configured WaveNet (networks.py:147,175-176); 255 for the shipped options. */
int lsph_receptive_field(lsph_handle h, int* out);

/* Introspection (tests; works on a host-only handle): the arrays lsph_load_weights packed, as the kernels read them.
 * which: 0 w_fg [L][2R][2R] (filter rows then gate rows; tap 0 = x[t-d] half, tap 1 = x[t] half), 1 w_rs [L][R+S][R]
 * (residual_conv rows then skip_conv rows), 2 b_rs [L][R+S], 3 w_cond [L*2R][cond_ch], 4 b_cond [L*2R] (cond conv bias +
 * filter/gate conv bias), 5 / 6 scale / shift [apc_hidden] of the BatchNorm-folded first linear layer. */
int lsph_debug_packed(lsph_handle h, int which, float* dst, int64_t count);

int lsph_destroy(lsph_handle h);
const char* lsph_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* LSPH_H_ */
