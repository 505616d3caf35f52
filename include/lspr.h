/*
 * lspr.h - C ABI of the H100-native recurrent audio networks of LiveSpeechPortraits (demo.py stages 1 and 3).
 *
 * What it replaces:
 *   LSPR_APC    APC_encoder.forward (models/networks.py:20-69; demo.py:186-192): a stack of single-layer GRUs,
 *               mel_dim -> hidden -> ... -> hidden, over every mel frame of a clip (batch 1, full length).
 *   LSPR_MOUTH  Audio2Feature.forward with feature_decoder='LSTM' (models/audio2feature.py:32-69) as
 *               Audio2FeatureModel.generate_sequences drives it (models/audio2feature_model.py:117-154): downsample MLP
 *               over pairs of APC rows, a 3-layer LSTM with 256 units, then the fc MLP on the frames that are kept.
 *
 * Every layer's input projection X W_ih^T + b is one fp32 GEMM over all time steps; the recurrence of a layer is one
 * persistent launch of a single thread-block cluster whose CTAs each keep their hidden units' rows of W_hh in shared
 * memory and exchange h_t through distributed shared memory, one cluster barrier per step (see csrc/lspr.cu).
 * All arithmetic is fp32 with a fixed summation order: repeated runs are bit-identical.
 *
 * Conventions as in lspg.h: plain C types, 0 or a negative LSPG_E* code, message in lspr_last_error(); sm_90 only,
 * no CPU path.  The Python binding is livespeechportraits_b200/recurrent.py.
 */
#ifndef LSPR_H_
#define LSPR_H_

#include <stddef.h>
#include <stdint.h>

#include "lspg.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct lspr_ctx* lspr_handle;

enum { LSPR_APC = 0, LSPR_MOUTH = 1 };

/* The option fields the two modules' constructors read. */
typedef struct lspr_config {
  int kind;          /* LSPR_APC or LSPR_MOUTH */
  int input_dim;     /* APC: mel_dim (80), a multiple of 16.  MOUTH: APC_hidden_size (512), a multiple of 64 */
  int hidden;        /* APC: hidden_size, must be 512.  MOUTH: ignored (the LSTM has 256 units, models/audio2feature.py:40) */
  int num_layers;    /* APC: num_layers (3), 1..8.  MOUTH: ignored (3 layers) */
  int residual;      /* APC: residual (config/<id>.yaml; false for the shipped configs).  MOUTH: ignored */
  int frame_future;  /* MOUTH: frame_future (18), >= 0.  APC: ignored */
  int out_dim;       /* MOUTH: output size of the last fc layer ((2 A2L_GMM_ndim + 1) ncenter or A2L_GMM_ndim
                        predict_length; 75 shipped), 1..4096.  APC: ignored */
} lspr_config;

/* device == -1: host-only handle (weight packing introspection; lspr_forward returns LSPG_ENODEV). */
int lspr_create(lspr_handle* out, const lspr_config* cfg, int device);

/* Replaces load_state_dict.  Keys as in the reference module's state_dict(), optional "module." prefix, host fp32:
 *   APC    rnns.{i}.weight_ih_l0, rnns.{i}.weight_hh_l0, rnns.{i}.bias_ih_l0, rnns.{i}.bias_hh_l0
 *   MOUTH  downsample.{0,3}.{weight,bias}, downsample.1.{weight,bias,running_mean,running_var},
 *          LSTM.{weight_ih,weight_hh,bias_ih,bias_hh}_l{k}, fc.{0,3,6}.{weight,bias}, fc.{1,4}.{weight,bias,running_mean,running_var}
 * num_batches_tracked and unknown keys are ignored; every listed parameter must be present.  Eval-mode BatchNorm1d
 * (eps 1e-5) is folded into the preceding linear layer's epilogue as a per-channel scale and shift. */
int lspr_load_weights(lspr_handle h, const lspg_tensor* tensors, int n);

/* Bytes of device workspace lspr_forward needs for n_rows input rows. */
int lspr_workspace_bytes(lspr_handle h, int n_rows, size_t* bytes);

/* DEVICE pointers, fp32, contiguous, 16-byte aligned:
 *   APC    in [n_rows, input_dim] mel frames                -> out [n_rows, hidden]   (n_rows >= 0)
 *   MOUTH  in [n_rows, input_dim] APC features, n_rows even -> out [n_rows / 2, out_dim]   (n_rows >= 2)
 * ws: lspr_workspace_bytes(h, n_rows) bytes, 256-byte aligned.  cluster: CTAs per recurrence launch, 0 = library
 * choice (APC: 16 when a 16-CTA cluster can be scheduled, else 8 with part of W_hh read from L2; MOUTH: 8); APC accepts
 * 8 or 16, MOUTH 8.  Asynchronous on `stream`. */
int lspr_forward(lspr_handle h, const float* in, int n_rows, float* out, void* ws, size_t ws_bytes, int cluster, void* stream);

/* Introspection (tests; works on a host-only handle): the arrays lspr_load_weights packed, as the kernels read them.
 * G = 3 (GRU: r, z, n) or 4 (LSTM: i, f, g, o), H = hidden units of the layer, In = its input width.  Gate rows are
 * interleaved by unit: packed row u*G + g is torch's row g*H + u, so the rows of units [c*H/CL, (c+1)*H/CL) - those
 * CTA c of a CL-CTA cluster keeps - are one contiguous block for every CL.
 *   which = 4*l + 0   w_ih [G*H][In] of recurrent layer l
 *           4*l + 1   b    [G*H]  b_ih + b_hh (GRU n gate: b_in only)
 *           4*l + 2   w_hh [G*H][H]
 *           4*l + 3   b_hn [H] (GRU; zero-length for the LSTM)
 *   MOUTH, after the 3 LSTM layers (which = 12 + 3*s + {0: weight [N][K], 1: scale [N], 2: shift [N]}) the five linear
 *           stages s = downsample.0 (BN folded), downsample.3, fc.0 (BN), fc.3 (BN), fc.6; LeakyReLU follows stages 0, 2, 3.
 * dst == NULL: *count receives the element count.  Otherwise *count must equal it. */
int lspr_debug_packed(lspr_handle h, int which, float* dst, int64_t* count);

int lspr_destroy(lspr_handle h);
const char* lspr_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* LSPR_H_ */
