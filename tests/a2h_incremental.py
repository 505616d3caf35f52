"""Host emulator of the INCREMENTAL form of the Audio2Headpose loop, exactly as csrc/headpose.cuh runs it: one new time
step per generated frame, per-layer activation history instead of a full 255-step WaveNet forward per frame.

Why it is the same function as the reference loop (models/audio2headpose_model.py:169-187): the receptive field of the
last output position equals the window length (255), so the cone of activations that feed output position 254 of window i
never touches the zero padding of that window; every activation in the cone is a function of absolute-time inputs only and
is identical in every window that contains it.  So: run the recurrence over absolute time t = 0 .. rf-2+nframe, where the
first rf-1 steps replay window 0 (history = pre_headpose, audio = first row repeated; taps that reach before t = 0 read the
zero padding of window 0) and step t = i + rf - 1 produces frame i.  tests/test_a2h_oracle.py checks this against the oracle.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import a2h_oracle as A


def lrelu(x):
    return np.where(x > 0, x, 0.2 * x)


def generate_incremental(sd, audio_feats, pre_headpose, noise, opt, sigma_scale=0.3, return_params=False):
    f64 = lambda k: sd[k].double().numpy()      # noqa: E731  float64 emulation: isolates algorithmic equivalence from rounding
    bias = lambda k, n: f64(k) if k in sd else np.zeros(n)     # noqa: E731  conv biases are absent when use_bias is off
    ff, rf = opt.frame_future, opt.A2H_receptive_field
    ndim, nc = opt.A2H_GMM_ndim, opt.A2H_GMM_ncenter
    audio = np.asarray(audio_feats, np.float64).reshape(-1, 2 * opt.APC_hidden_size)
    n_audio = audio.shape[0]
    nframe = n_audio - ff
    dil = A.dilations(opt)
    nl = len(dil)
    # ---- precompute (not autoregressive): audio_downsample of every row, cond projections of every block
    with torch.no_grad():
        ds = A.audio_downsample({k: v.double() for k, v in sd.items() if k.startswith("audio_downsample") and v.dtype.is_floating_point},
                                torch.from_numpy(audio)).numpy()
    cf = [ds @ f64(f"WaveNet.residual_blocks.{i}.cond_filter_conv.weight")[:, :, 0].T + f64(f"WaveNet.residual_blocks.{i}.cond_filter_conv.bias") for i in range(nl)]
    cg = [ds @ f64(f"WaveNet.residual_blocks.{i}.cond_gate_conv.weight")[:, :, 0].T + f64(f"WaveNet.residual_blocks.{i}.cond_gate_conv.bias") for i in range(nl)]
    W1, b1 = f64("WaveNet.start_conv1.weight")[:, :, 0], f64("WaveNet.start_conv1.bias")
    W2, b2 = f64("WaveNet.start_conv2.weight")[:, :, 0], f64("WaveNet.start_conv2.bias")
    E1, e1 = f64("WaveNet.end_conv_1.weight")[:, :, 0], f64("WaveNet.end_conv_1.bias")
    E2, e2 = f64("WaveNet.end_conv_2.weight")[:, :, 0], f64("WaveNet.end_conv_2.bias")
    blk = []
    for i in range(nl):
        p = f"WaveNet.residual_blocks.{i}."
        R_, S_ = opt.A2H_wavenet_residual_channels, opt.A2H_wavenet_skip_channels
        blk.append(dict(Wf=f64(p + "filter_conv.weight"), bf=bias(p + "filter_conv.bias", R_), Wg=f64(p + "gate_conv.weight"),
                        bg=bias(p + "gate_conv.bias", R_), Wr=f64(p + "residual_conv.weight")[:, :, 0], br=bias(p + "residual_conv.bias", R_),
                        Ws=f64(p + "skip_conv.weight")[:, :, 0], bs=bias(p + "skip_conv.bias", S_)))
    T = rf - 1 + nframe
    R = opt.A2H_wavenet_residual_channels
    X = np.zeros((nl, T, R))                        # input of block l at absolute time t
    h = np.asarray(pre_headpose, np.float64).copy()
    pred = np.zeros((nframe, ndim))
    params = np.zeros((nframe, A.output_size(opt)))
    for t in range(T):
        r = min(max(t + ff - (rf - 1), 0), n_audio - 1)          # audio row whose features condition absolute time t
        x = lrelu(W2 @ lrelu(W1 @ h + b1) + b2)
        emit = t >= rf - 1
        skip = np.zeros(opt.A2H_wavenet_skip_channels)
        for l, d in enumerate(dil):
            X[l, t] = x
            xd = X[l, t - d] if t - d >= 0 else np.zeros(R)       # zero padding of window 0 (networks.py:307)
            B = blk[l]
            f = B["Wf"][:, :, 0] @ xd + B["Wf"][:, :, 1] @ x + B["bf"] + cf[l][r]
            g = B["Wg"][:, :, 0] @ xd + B["Wg"][:, :, 1] @ x + B["bg"] + cg[l][r]
            z = np.tanh(f) * (1.0 / (1.0 + np.exp(-g)))
            if emit:
                skip += B["Ws"] @ z + B["bs"]
            x = B["Wr"] @ z + B["br"] + x
        if emit:
            i = t - (rf - 1)
            out = E2 @ lrelu(E1 @ lrelu(skip) + e1) + e2
            params[i] = out
            if opt.loss == "GMM":
                mu = out[nc:nc + ndim]                             # ncenter == 1: component 0
                sigma = np.exp(-out[nc + nc * ndim:nc + nc * ndim + ndim]) * sigma_scale
                h = noise[i].astype(np.float64) * sigma + mu
            else:
                h = out[:ndim]
            pred[i] = h
    return (pred, params) if return_params else pred
