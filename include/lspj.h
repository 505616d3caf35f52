/*
 * lspj.h - C ABI of the H100-native baseline JPEG encoder.
 *
 * What it replaces: demo.py's JPEG boundary - visualizer.save_images writes every predicted frame (and every feature map)
 * through util.save_image, which is PIL's Image.save(path) at its defaults: quality 75, 4:2:0, baseline, standard Huffman
 * tables.  Here the frames never leave the device as raw pixels: each slot of `out` receives the complete .jpg file PIL
 * (libjpeg-turbo) writes for the same uint8 image, byte for byte.
 *
 * The arithmetic is libjpeg-turbo's baseline path as PIL drives it: jpeg_quality_scaling with force_baseline (tables
 * clamped to 1..255), rgb_ycc_convert's 16-bit fixed point, h2v2_downsample with the alternating 1/2 bias, jfdctint
 * (islow: CONST_BITS 13, PASS1_BITS 2), quantize's divide by 8 * table rounded half away from zero, jchuff's standard
 * tables (ZRL only before a nonzero coefficient, EOB after trailing zeros, negative magnitudes written as v - 1),
 * per-component DC prediction in MCU order (Y0 Y1 Y2 Y3 Cb Cr), 0xFF -> 0xFF 0x00 stuffing (the final 1-bit padding
 * included) and jcmarker's segments: SOI, JFIF APP0 1.01 (no units, 1:1), one DQT per table, SOF0, one DHT per table
 * (DC 0, AC 0, DC 1, AC 1), SOS, scan, EOI.  oracle/jpeg_oracle.py restates each stage in numpy.
 *
 * The bound lspj_max_bytes.  Per 8x8 block the coded scan holds at most
 *   DC:  one code of at most 16 bits + at most 11 magnitude bits (|diff| <= 2047 for 8-bit samples)        27
 *   AC:  63 codes of at most 16 bits, each with at most 10 magnitude bits (|coef| <= 1023)           63 * 26 = 1638
 *   ZRL: at most 3 (a ZRL stands for 16 zeros and precedes a nonzero coefficient; 63 / 16 < 4), 16 bits    48
 *   EOB: at most one, 16 bits                                                                               16
 * = B = 1729 bits.  A frame of N blocks (N = H W / 64 grey, 6 H W / 256 colour) has a scan of at most
 * S = ceil(N B / 8) bytes including the 1-bit padding, at most one stuffed 0x00 per scan byte, so the file is at most
 * header + 2 S + 2 (EOI) bytes; the header is 623 bytes in colour and 328 in grey.
 *
 * Conventions as in lspg.h / lspa.h: plain C types, 0 or a negative LSPG_E* code, message in lspj_last_error(); sm_90
 * only, no CPU path.  The Python binding is livespeechportraits_b200/jpeg.py.
 */
#ifndef LSPJ_H_
#define LSPJ_H_

#include <stddef.h>
#include <stdint.h>

#include "lspg.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct lspj_ctx* lspj_handle;

/* device == -1: host-only handle (argument checking and sizes only; lspj_encode returns LSPG_ENODEV). */
int lspj_create(lspj_handle* out, int device);

/* The bound derived above for one file of a height x width frame with `components` (1 grey, 3 RGB) channels.
 * LSPG_EINVAL unless height and width are multiples of 16 in [16, 65535], components is 1 or 3, and the bound is at
 * most 2^30 bytes. */
int lspj_max_bytes(lspj_handle h, int height, int width, int components, size_t* bytes);

/* Device workspace of lspj_encode for n such frames (n >= 0); the same argument checks. */
int lspj_workspace_bytes(lspj_handle h, int n, int height, int width, int components, size_t* bytes);

/* Encodes n frames at `quality` (1..100).  images: device uint8, 16-byte aligned, [n][height][width][3] RGB (components
 * 3) or [n][height][width] grey (components 1).  out: device, n slots of out_stride >= lspj_max_bytes bytes; slot i
 * receives frame i's complete .jpg file and sizes[i] (device int32 [n]) its length.  ws: device, 256-byte aligned, at
 * least lspj_workspace_bytes.  Asynchronous on `stream`; allocates nothing and does not synchronise the host.  Calls on
 * different streams with different workspaces run independently.  n == 0 launches nothing. */
int lspj_encode(lspj_handle h, const uint8_t* images, int n, int height, int width, int components, int quality,
                uint8_t* out, int64_t out_stride, int32_t* sizes, void* ws, size_t ws_bytes, void* stream);

int lspj_destroy(lspj_handle h);
const char* lspj_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* LSPJ_H_ */
