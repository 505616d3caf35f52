/*
 * lspa.h - C ABI of the H100-native log-mel front end (LiveSpeechPortraits, SURVEY.md 8f row N6).
 *
 * What it replaces: stage 1 of demo.py (:185) - funcs/utils.py compute_mel_one_sequence (:61-83), a Python loop that
 * for each of 2 nframe windows copies a 266-sample clip to the device, runs Audio2Mel.forward (funcs/audio_funcs.py:56-75:
 * reflect pad, one torch.stft frame, sqrt, an [80, 257] matmul, log) and copies the 80 values back.  Here one kernel
 * computes every window of the clip.
 *
 * Conventions as in lspg.h / lspm.h: plain C types, 0 or a negative LSPG_E* code, message in lspa_last_error(); sm_90
 * only, no CPU path.  lspa_logmel_at is asynchronous on `stream` and allocates nothing.  The Python binding is
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

/* device == -1: host-only handle (argument checking only; lspa_load_mel_basis / lspa_logmel_at return LSPG_ENODEV). */
int lspa_create(lspa_handle* out, int device);

/* Audio2Mel.mel_basis: host fp32 [n_mels, n_bins], 1 <= n_mels <= 128, n_bins == 257 (n_fft 512).  Synchronous: copies
 * to a library-owned device buffer.  A second call replaces the basis. */
int lspa_load_mel_basis(lspa_handle h, const float* host_basis, int n_mels, int n_bins);

/* compute_mel_one_sequence with the loaded basis, on the whole clip or a piece of it.  audio: device fp32 [n_samples],
 * any alignment (may be NULL when n_samples == 0), holding the clip's samples [first_sample, first_sample + n_samples).
 * out: device fp32 [n_windows, n_mels], receiving windows first_window .. first_window + n_windows - 1.  Window i
 * (i the index in the whole clip) is the clip audio[st : st + frame_len] with st = (int64_t)(i * step) (an fp64 product,
 * truncated), 190 <= frame_len <= 266; it is reflect-padded by 189, multiplied by the periodic Hann window of 266 centred
 * in 512, and its 257-bin magnitude spectrum is mapped through the basis: out[i][m] = log(max(sum_k basis[m][k] |X_k|,
 * 1e-5)), and with normalize != 0 (out - log(1e-5)) / -log(1e-5) in fp32.  Samples at or past first_sample + n_samples
 * read as zero, which is the clip's end padding, so a streaming caller passes a window that reaches past the samples it
 * has only once the clip has ended; each row depends only on its window, so a piece's rows are bit-identical to the same
 * rows of the whole clip.  The whole clip is first_sample = 0, first_window = 0.  LSPG_EINVAL when window first_window
 * starts before first_sample, or for first_sample < 0, first_window < 0 or first_window + n_windows >= 2^31.
 * n_windows == 0 launches nothing. */
int lspa_logmel_at(lspa_handle h, const float* audio, int64_t first_sample, int64_t n_samples, int first_window,
                   int n_windows, int frame_len, double step, int normalize, float* out, void* stream);

/* The resampling step of librosa.load (resampy.resample with a kaiser table, then resample_f), from native-rate frames
 * to the rate sample_ratio * orig_sr.
 *
 * lspa_load_resample_filter: the filter for one sample_ratio = float(sr_new) / sr_orig, as resampy hands it to
 * resample_f: host fp64 win[nwin] (the half window, already multiplied by sample_ratio when sample_ratio < 1), delta[nwin]
 * (win[j + 1] - win[j], delta[nwin - 1] = 0) and num_table (table entries per zero crossing, 2^precision).  Synchronous:
 * copies to a library-owned device buffer; a second call replaces the filter. */
int lspa_load_resample_filter(lspa_handle h, const double* win, const double* delta, int nwin, int num_table,
                              double sample_ratio);

#define LSPA_FMT_F32 0 /* float32 samples */
#define LSPA_FMT_S16 1 /* PCM16 samples, decoded as s / 32768 */

/* Outputs first_out .. first_out + n_out - 1 of a clip into out (device fp32 [n_out]), with the loaded filter.
 * frames: device [n_in, channels] interleaved (format LSPA_FMT_F32 or LSPA_FMT_S16, channels 1 or 2) holding the clip's
 * frames [first_in, first_in + n_in); each frame is decoded and mixed to mono as librosa.load does (fp32 (c0 + c1) / 2).
 * Frames outside the buffer read as zero: before frame 0 and after the clip's end that is what the reference's wing
 * clamps compute, so the arithmetic does not depend on the clip's length, only the output count does
 * (int(n * sample_ratio)).  reg_table: host int64 [n_reg][4], the time register of output t in closed form per binade:
 * row {t_b, base, k, e} gives register(t) = (base + (t - t_b) * k) * 2^e for t_b <= t < the next row's t_b; row 0 starts
 * at t_b = 0 and the last row {t_end, 0, 0, 0} ends the table, which must reach first_out + n_out.  Output t is
 * resample_f's sum over the left wing, then the right wing, each tap an fp64 product and sum rounded to fp32.
 * LSPG_EINVAL for bad counts, formats or channels, a malformed table, or first_in > 0 when output first_out's left wing
 * can read before first_in (n - (nwin / index_step - 1) < first_in, n = (int64_t)register(first_out)).  Asynchronous on
 * `stream`; allocates nothing. */
int lspa_resample_at(lspa_handle h, const void* frames, int format, int channels, int64_t first_in, int64_t n_in,
                     int64_t first_out, int64_t n_out, const int64_t* reg_table, int n_reg, float* out, void* stream);

int lspa_destroy(lspa_handle h);
const char* lspa_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* LSPA_H_ */
