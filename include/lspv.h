/*
 * lspv.h - C ABI of the H100-native H.264 encoder.
 *
 * What it is for: the reference writes its videos inter-coded (demo.py: DIVX through cv2, predict.py: H.264 MP4 through
 * ffmpeg), and a live session needs a stream small enough to send.  The H100 has no NVENC, so this module encodes on
 * the SMs: uint8 frames on the device in, Annex B access units on the device out, no host synchronisation.  There is no
 * canonical H.264 encoder to match; the contract is that every access unit decodes, in any conforming decoder, to
 * exactly the reconstruction the encoder keeps in its state (H.264 defines decoding bit for bit, and this subset has no
 * loop filter).  oracle/h264_oracle.py restates each stage in numpy.
 *
 * The bitstream: one fixed subset of Constrained Baseline.
 *   SPS  profile_idc 66, constraint_set0/1 set, level_idc the lowest of Table A-1 whose MaxFS, MaxMBPS (fps x frame
 *        macroblocks), MaxDpbMbs (one frame) and sqrt(8 MaxFS) frame-dimension limit hold (bit rate is not
 *        constrained), log2_max_frame_num 4, pic_order_cnt_type 2, one reference frame, frame_mbs_only, no cropping
 *        (H and W are multiples of 16).  VUI: video_format 5, limited range, colour primaries / transfer / matrix 6
 *        (SMPTE 170M, BT.601), timing num_units_in_tick 1, time_scale 2 fps, fixed_frame_rate; bitstream_restriction
 *        with max_num_reorder_frames 0 and max_dec_frame_buffering 1, so decoders output every frame at once.
 *   PPS  CAVLC, one slice group, one reference index, pic_init_qp 26, chroma_qp_index_offset 0, deblocking filter
 *        control present.
 *   Access unit f: IDR when f % gop == 0 (start code + SPS, start code + PPS, start code + IDR slice, nal_ref_idc 3),
 *        else one P slice (nal_ref_idc 3).  4-byte start codes; 00 00 0x (x <= 3) -> 00 00 03 0x in every NAL unit.
 *   Slice header: first_mb 0, slice_type 7 (I) / 5 (P), frame_num (f % gop) % 16, idr_pic_id (f / gop) & 1,
 *        slice_qp_delta QP - 26, disable_deblocking_filter_idc 1.  mb_qp_delta is always 0.
 *
 * Colour (integer, >> is a floor shift):
 *   Y  = ((66 R + 129 G + 25 B + 128) >> 8) + 16
 *   Cb = ((-38 R - 74 G + 112 B + 128) >> 8) + 128,  Cr = ((112 R - 94 G - 18 B + 128) >> 8) + 128 per pixel, then
 *   4:2:0 as (sum of the 2x2 + 2) >> 2.  Grey input g is R = G = B = g (Cb = Cr = 128).
 *
 * I frames: every macroblock I_16x16.  Luma modes V (0), H (1), DC (2), Plane (3) and chroma modes DC (0), H (1),
 *   V (2), Plane (3), each only where its neighbours exist (8.3.3, 8.3.4); the least SAD of source - prediction wins
 *   (chroma: Cb's + Cr's), the lower mode number on ties.  Prediction reads the reconstructed left, top and top-left
 *   neighbours, so macroblock (x, y) waits for (x - 1, y) and (x, y - 1): a wavefront of macroblock rows.
 * P frames: every macroblock P_L0_16x16 or P_Skip, never intra.  A full-pel vector (dx, dy) with |dx|, |dy| <= search
 *   and the 16x16 block inside the frame minimises SAD + lambda[QP] (se bits of 4 dx + se bits of 4 dy) - the vector's
 *   cost coded from zero, so every macroblock decides on its own; ties go to the smaller dy, then the smaller dx.
 *   lambda[QP] = round(sqrt(0.85 x 2^((QP - 12) / 3))):
 *     0 0 0 0 0 0 0 1 1 1 1 1 1 1 1 1 1 2 2 2 2 3 3 3 4 4 5 5 6 7 7 8 9 10 12 13 15 17 19 21 23 26 30 33 37 42 47 53 59
 *     66 74 83.
 *   Luma prediction is the reference block itself; chroma uses 8.4.2.2.2's eighth-sample bilinear filter with edge
 *   clamping (an odd dx or dy is a half-sample chroma vector).  A macroblock is P_Skip when its vector equals 8.4.1.1's
 *   P_Skip vector and all its levels are zero; otherwise its mvd is coded against 8.4.1.3's median prediction.
 * Residual: the forward core transform Cf X Cf^T per 4x4 block; the I_16x16 luma DCs take (H D H) >> 1 (H the 4x4
 *   Hadamard), the chroma DCs the 2x2 transform.  Level = sign(W) ((|W| MF + f) >> qbits), qbits = 15 + QP / 6, MF the
 *   standard multipliers (13107 5243 8066 / 11916 4660 7490 / 10082 4194 6554 / 9362 3647 5825 / 8192 3355 5243 /
 *   7282 2893 4559 for positions (even, even), (odd, odd), other), f = 2^qbits / 3 intra and 2^qbits / 6 inter
 *   (integer division); DC blocks use MF(0, 0), 2 f and qbits + 1.  Chroma uses Table 8-15's QPc.  Levels are clamped
 *   to +-2063, the largest magnitude CAVLC codes with level_prefix <= 15 under every suffixLength.  Scaling and the
 *   inverse transforms are 8.5.10-8.5.12 with flat scaling lists.
 * CAVLC: coeff_token with nC from the neighbours' TotalCoeff (chroma DC nC = -1), trailing-one signs, levels with the
 *   suffixLength adaptation and the level_prefix 14 / 15 escapes, total_zeros, run_before; mb_skip_run,
 *   coded_block_pattern through Table 9-4's inter mapping, I_16x16 mb_type carrying mode and cbp.  I_16x16 luma cbp is
 *   15 when any AC level is nonzero; chroma cbp is 2 with any chroma AC level, 1 with only DC levels.
 *
 * The bound lspv_max_bytes.  A 4x4 block of N <= 16 levels codes in at most 16 (coeff_token) + 28 N (a level:
 *   level_prefix <= 16 bits + a 12-bit suffix) + 9 (total_zeros) + 11 (N - 1) (run_before) bits; a chroma DC block in
 *   8 + 4 x 28 + 3 + 3 x 2 = 129.  Then a macroblock is at most
 *     I_16x16:    9 (mb_type) + 5 (chroma mode) + 1 (qp delta) + B(16) + 16 B(15) + 2 x 129 + 8 B(15)  = 15258 + 29
 *     P_L0_16x16: 1 + 2 x 21 (|mvd| <= 8 x 64 quarter samples) + 11 (cbp) + 1 + 16 B(16) + 2 x 129 + 8 B(15) = 15313
 *   bits, plus at most one mb_skip_run code of ue(M) for M macroblocks.  The access unit is at most 2 x 64 bytes of
 *   parameter sets, 5 bytes of start code and NAL header, and an RBSP of R = ceil((64 + M x MB + 8) / 8) bytes with at
 *   most one emulation-prevention byte per two: 133 + R + ceil(R / 2).
 *
 * State (lspv_state_bytes, caller-owned, 256-byte aligned): int64 index of the next frame, then at byte 256 the last
 * reconstructed frame as Y [H][W], Cb [H/2][W/2], Cr [H/2][W/2] uint8.  A call encodes frames f0 .. f0 + n - 1 from the
 * state the call that ended at f0 left (any state when f0 % gop == 0): a whole clip is one call from f0 = 0, a live
 * session one call per push, and the two give the same bytes.
 *
 * Conventions as in lspg.h / lspj.h: plain C types, 0 or a negative LSPG_E* code, message in lspv_last_error(); sm_90
 * only, no CPU path.  The Python binding is livespeechportraits_b200/h264.py.
 */
#ifndef LSPV_H_
#define LSPV_H_

#include <stddef.h>
#include <stdint.h>

#include "lspg.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct lspv_ctx* lspv_handle;

/* qp 0..51, gop >= 1 (IDR period), search 0..64 (full-pel range), fps 1..1000.  device == -1: host-only handle
 * (argument checking and sizes only; lspv_encode returns LSPG_ENODEV). */
int lspv_create(lspv_handle* out, int qp, int gop, int search, int fps, int device);

/* The bound derived above for one access unit of a height x width frame.  LSPG_EINVAL unless height and width are
 * multiples of 16 in [16, 65535], some level holds the frame at the handle's fps, and the bound is at most 2^30. */
int lspv_max_bytes(lspv_handle h, int height, int width, size_t* bytes);

/* Bytes of the caller-owned encoder state for that frame size; the same argument checks. */
int lspv_state_bytes(lspv_handle h, int height, int width, size_t* bytes);

/* Device workspace of lspv_encode for that frame size (any number of frames); the same argument checks. */
int lspv_workspace_bytes(lspv_handle h, int height, int width, size_t* bytes);

/* Encodes frames f0 .. f0 + n - 1.  images: device uint8 [n][height][width][3] RGB (components 3) or [n][height][width]
 * grey (components 1).  state: see above.  out: device, n slots of out_stride >= lspv_max_bytes bytes; slot i receives
 * access unit f0 + i, sizes[i] (device int32) its length and is_idr[i] (device uint8) 1 for an IDR.  ws: device,
 * 256-byte aligned, at least lspv_workspace_bytes.  Frames run in order on `stream`, asynchronously; nothing is
 * allocated and the host is not synchronised.  n == 0 launches nothing. */
int lspv_encode(lspv_handle h, const uint8_t* images, int n, int height, int width, int components, int64_t f0,
                void* state, uint8_t* out, int64_t out_stride, int32_t* sizes, uint8_t* is_idr, void* ws,
                size_t ws_bytes, void* stream);

int lspv_destroy(lspv_handle h);
const char* lspv_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* LSPV_H_ */
