/*
 * lspa.h - C ABI of the H100-native log-mel front end (LiveSpeechPortraits, SURVEY.md 8f row N6).
 *
 * What it replaces: stage 1 of demo.py (:185) - funcs/utils.py compute_mel_one_sequence (:61-83), a Python loop that
 * for each of 2 nframe windows copies a 266-sample clip to the device, runs Audio2Mel.forward (funcs/audio_funcs.py:56-75:
 * reflect pad, one torch.stft frame, sqrt, an [80, 257] matmul, log) and copies the 80 values back.  Here one kernel
 * computes every window of the clip.
 *
 * Conventions as in lspg.h / lspm.h: plain C types, 0 or a negative LSPG_E* code, message in lspa_last_error(); sm_90
 * only, no CPU path.  lspa_logmel is asynchronous on `stream` and allocates nothing.  The Python binding is
 * livespeechportraits_b200/audio.py.
 */
#ifndef LSPA_H_
#define LSPA_H_

#include <stddef.h>
#include <stdint.h>

#include "lspg.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct lspa_ctx* lspa_handle;

/* device == -1: host-only handle (argument checking only; lspa_load_mel_basis / lspa_logmel return LSPG_ENODEV). */
int lspa_create(lspa_handle* out, int device);

/* Audio2Mel.mel_basis: host fp32 [n_mels, n_bins], 1 <= n_mels <= 128, n_bins == 257 (n_fft 512).  Synchronous: copies
 * to a library-owned device buffer.  A second call replaces the basis. */
int lspa_load_mel_basis(lspa_handle h, const float* host_basis, int n_mels, int n_bins);

/* compute_mel_one_sequence with the loaded basis.  audio: device fp32 [n_samples], any alignment (may be NULL when
 * n_samples == 0).  Window i (0 <= i < n_windows, n_windows < 2^31) is the clip audio[st : st + frame_len] with
 * st = (int64_t)(i * step) (an fp64 product, truncated), zero-padded past n_samples, 190 <= frame_len <= 266; it is
 * reflect-padded by 189, multiplied by the periodic Hann window of 266 centred in 512, and its 257-bin magnitude spectrum
 * is mapped through the basis: out[i][m] = log(max(sum_k basis[m][k] |X_k|, 1e-5)), and with normalize != 0
 * (out - log(1e-5)) / -log(1e-5) in fp32.  out: device fp32 [n_windows, n_mels].  n_windows == 0 launches nothing. */
int lspa_logmel(lspa_handle h, const float* audio, int64_t n_samples, int n_windows, int frame_len, double step,
                int normalize, float* out, void* stream);

int lspa_destroy(lspa_handle h);
const char* lspa_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* LSPA_H_ */
