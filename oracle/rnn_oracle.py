"""Oracle of the recurrent audio networks (include/lspr.h): the APC encoder (``APC_encoder``, models/networks.py:20-69)
and Audio2Mouth (``Audio2Feature`` with the LSTM decoder, models/audio2feature.py:32-69, driven by
``Audio2FeatureModel.generate_sequences``, models/audio2feature_model.py:117-154).  TEST INFRASTRUCTURE.

* Restatement (fp32, torch modules, the reference's arithmetic): ``apc_reference`` reuses ``mel_oracle.ApcGru``;
  ``Audio2MouthLSTM`` and ``generate_sequences`` restate the LSTM path.  oracle/make_golden_rnn.py checks both bit-equal
  against the unmodified reference code and writes tests/golden/rnn/.
* Float64 truth (``apc_truth``, ``mouth_truth``): the explicit gate equations and an exact eval-mode BatchNorm in float64,
  on the fp32 weights and inputs.  Runs on any torch device (the 10-minute case uses the GPU's float64 units).
* Emulator (``emulate_apc``, ``emulate_mouth``): the kernel's recurrence in float64, reading only the arrays
  ``lspr_load_weights`` packed - gate rows interleaved by unit, W_hh taken CTA slice by CTA slice, b_hn inside the n gate,
  BatchNorm as the folded scale / shift, the frame_future rows by clamping - so a packing mistake shows up on the host.
* Weight recipes: "A" torch's default initialisation; "B" the same with W_hh x 2 and the recurrent biases N(0, 0.5), so
  gates saturate and the state carries long memory.  In both, the BatchNorm layers get non-trivial running statistics
  and affine parameters (default ones would make the fold an identity).
"""
from __future__ import annotations

import types
from collections import OrderedDict
from typing import Dict

import numpy as np
import torch

from oracle.mel_oracle import ApcGru

LSTM_H = 256
BN_EPS = 1e-5


# ------------------------------------------------------------------------------------------------------------------
# Weights and inputs
# ------------------------------------------------------------------------------------------------------------------
def _recipe_b(sd: Dict[str, torch.Tensor], seed: int) -> None:
    g = torch.Generator().manual_seed(1000 + seed)
    for k, v in sd.items():
        if "weight_hh" in k:
            v.mul_(2.0)
        elif "bias_ih" in k or "bias_hh" in k:
            v.copy_(torch.randn(v.shape, generator=g) * 0.5)


def make_apc_state_dict(recipe: str = "A", seed: int = 0, mel_dim: int = 80, hidden: int = 512, layers: int = 3):
    """State dict of ``APC_encoder(mel_dim, hidden, layers)`` (keys ``rnns.{i}.weight_ih_l0``, ...)."""
    sd = OrderedDict((k, v.detach().clone()) for k, v in ApcGru(mel_dim, hidden, layers, seed).state_dict().items())
    if recipe == "B":
        _recipe_b(sd, seed)
    elif recipe != "A":
        raise ValueError(recipe)
    return sd


def default_mouth_opt(**over):
    """The option fields Audio2Feature reads, at their shipped defaults (options/base_options_audio2feature.py)."""
    o = dict(feature_decoder="LSTM", loss="L2", APC_hidden_size=512, A2L_GMM_ndim=25 * 3, A2L_GMM_ncenter=1,
             predict_length=1, frame_future=18)
    o.update(over)
    return types.SimpleNamespace(**o)


def mouth_output_size(opt) -> int:
    if opt.loss == "GMM":
        return (2 * opt.A2L_GMM_ndim + 1) * opt.A2L_GMM_ncenter
    return opt.A2L_GMM_ndim * opt.predict_length


class Audio2MouthLSTM(torch.nn.Module):
    """``Audio2Feature`` with ``feature_decoder='LSTM'``: the same modules in the same order, the same forward."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        D = opt.APC_hidden_size
        self.downsample = torch.nn.Sequential(torch.nn.Linear(D * 2, D), torch.nn.BatchNorm1d(D), torch.nn.LeakyReLU(0.2),
                                              torch.nn.Linear(D, D))
        self.LSTM = torch.nn.LSTM(input_size=D, hidden_size=LSTM_H, num_layers=3, dropout=0, bidirectional=False,
                                  batch_first=True)
        self.fc = torch.nn.Sequential(torch.nn.Linear(LSTM_H, 512), torch.nn.BatchNorm1d(512), torch.nn.LeakyReLU(0.2),
                                      torch.nn.Linear(512, 512), torch.nn.BatchNorm1d(512), torch.nn.LeakyReLU(0.2),
                                      torch.nn.Linear(512, mouth_output_size(opt)))

    def forward(self, audio_features):
        bs, item_len, ndim = audio_features.shape
        audio_features = audio_features.reshape(bs, -1, ndim * 2)
        down = self.downsample(audio_features.reshape(-1, ndim * 2)).reshape(bs, int(item_len / 2), ndim)
        output, _ = self.LSTM(down)
        return self.fc(output.reshape(-1, LSTM_H)).reshape(bs, int(item_len / 2), -1)


def make_mouth_state_dict(opt, recipe: str = "A", seed: int = 0):
    """State dict of ``Audio2Feature(opt)`` (LSTM decoder) under ``recipe``."""
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        m = Audio2MouthLSTM(opt)
    sd = OrderedDict((k, v.detach().clone()) for k, v in m.state_dict().items())
    g = torch.Generator().manual_seed(2000 + seed)
    for bn in ("downsample.1", "fc.1", "fc.4"):
        n = sd[bn + ".weight"].numel()
        sd[bn + ".weight"] = 0.5 + torch.rand(n, generator=g)
        sd[bn + ".bias"] = 0.1 * torch.randn(n, generator=g)
        sd[bn + ".running_mean"] = 0.1 * torch.randn(n, generator=g)
        sd[bn + ".running_var"] = 0.5 + torch.rand(n, generator=g)
    if recipe == "B":
        _recipe_b(sd, seed)
    elif recipe != "A":
        raise ValueError(recipe)
    return sd


def make_mel(T: int, seed: int = 0, mel_dim: int = 80) -> np.ndarray:
    """Normalised-log-mel-like fp32 frames in [0, 1] with a slow drift, seeded."""
    rng = np.random.Generator(np.random.PCG64(seed))
    drift = 0.5 + 0.3 * np.sin(np.arange(T)[:, None] / 50.0 + np.arange(mel_dim)[None] / 7.0)
    return np.clip(drift + 0.2 * rng.standard_normal((T, mel_dim)), 0.0, 1.0).astype(np.float32)


def make_feats(n: int, seed: int = 0, dim: int = 512) -> np.ndarray:
    """APC-feature-like fp32 rows in (-1, 1), seeded."""
    rng = np.random.Generator(np.random.PCG64(seed))
    return np.tanh(rng.standard_normal((n, dim)) * 0.7).astype(np.float32)


# ------------------------------------------------------------------------------------------------------------------
# Restatement (fp32, the reference's arithmetic)
# ------------------------------------------------------------------------------------------------------------------
def apc_module(sd) -> ApcGru:
    layers = len([k for k in sd if k.endswith("weight_ih_l0")])
    m = ApcGru(sd["rnns.0.weight_ih_l0"].shape[1], sd["rnns.0.weight_hh_l0"].shape[1], layers)
    m.load_state_dict(sd)
    return m.eval()


@torch.no_grad()
def apc_reference(sd, mel, residual: bool = False) -> np.ndarray:
    """``APC_encoder.forward(mel[None], [T])[0]`` on the CPU in fp32.  With ``residual`` it is ``ApcGru.forward``;
    without, the same stack with no additions."""
    m = apc_module(sd)
    x = torch.as_tensor(np.asarray(mel, np.float32))
    if residual:
        return m(x).numpy()
    y = x[None]
    for rnn in m.rnns:
        y = rnn(y)[0]
    return y[0].numpy()


def mouth_module(opt, sd) -> Audio2MouthLSTM:
    m = Audio2MouthLSTM(opt)
    m.load_state_dict(sd)
    return m.eval()


def generate_sequences(module, audio_feats: np.ndarray, opt) -> np.ndarray:
    """models/audio2feature_model.py:130-154 restated: append 2 frame_future copies of the last row, forward, drop the
    first frame_future predictions."""
    frame_future = opt.frame_future
    nframe = int(audio_feats.shape[0] / 2)
    if not frame_future == 0:
        insert = np.repeat(audio_feats[-1], 2 * frame_future).reshape(-1, 2 * frame_future).T
        audio_feats = np.concatenate([audio_feats, insert])
    module.eval()
    with torch.no_grad():
        preds = module.forward(torch.from_numpy(audio_feats).unsqueeze(0).float())
    preds = preds[0, frame_future:].numpy() if frame_future else preds[0, :].numpy()
    assert preds.shape[0] == nframe
    return preds


# ------------------------------------------------------------------------------------------------------------------
# Float64 truth
# ------------------------------------------------------------------------------------------------------------------
def _t64(a, device):
    return torch.as_tensor(np.asarray(a) if not isinstance(a, torch.Tensor) else a).to(device=device, dtype=torch.float64)


@torch.no_grad()
def gru_layer_truth(x, w_ih, w_hh, b_ih, b_hh):
    """torch.nn.GRU's equations in the dtype of the inputs: x [T, In] -> h [T, H]."""
    H = w_hh.shape[1]
    gi = x @ w_ih.T + b_ih
    h = torch.zeros(H, dtype=x.dtype, device=x.device)
    out = torch.empty((x.shape[0], H), dtype=x.dtype, device=x.device)
    for t in range(x.shape[0]):
        gh = w_hh @ h + b_hh
        r = torch.sigmoid(gi[t, :H] + gh[:H])
        z = torch.sigmoid(gi[t, H:2 * H] + gh[H:2 * H])
        n = torch.tanh(gi[t, 2 * H:] + r * gh[2 * H:])
        h = (1 - z) * n + z * h
        out[t] = h
    return out


@torch.no_grad()
def lstm_layer_truth(x, w_ih, w_hh, b_ih, b_hh):
    """torch.nn.LSTM's equations (gates i, f, g, o): x [T, In] -> h [T, H]."""
    H = w_hh.shape[1]
    gi = x @ w_ih.T + b_ih + b_hh
    h = torch.zeros(H, dtype=x.dtype, device=x.device)
    c = torch.zeros_like(h)
    out = torch.empty((x.shape[0], H), dtype=x.dtype, device=x.device)
    for t in range(x.shape[0]):
        g = gi[t] + w_hh @ h
        i, f, gg, o = torch.sigmoid(g[:H]), torch.sigmoid(g[H:2 * H]), torch.tanh(g[2 * H:3 * H]), torch.sigmoid(g[3 * H:])
        c = f * c + i * gg
        h = o * torch.tanh(c)
        out[t] = h
    return out


@torch.no_grad()
def apc_truth(sd, mel, residual: bool = False, device="cpu") -> torch.Tensor:
    """Float64 APC features [T, hidden] on ``device``."""
    p = lambda k: _t64(sd[k], device)      # noqa: E731
    layers = len([k for k in sd if k.endswith("weight_ih_l0")])
    x = _t64(np.asarray(mel, np.float32), device)
    for i in range(layers):
        y = gru_layer_truth(x, p(f"rnns.{i}.weight_ih_l0"), p(f"rnns.{i}.weight_hh_l0"), p(f"rnns.{i}.bias_ih_l0"),
                            p(f"rnns.{i}.bias_hh_l0"))
        if residual and i + 1 < layers and y.shape[1] == x.shape[1]:
            y = y + x
        x = y
    return x


def _lrelu(x):
    return torch.where(x > 0, x, 0.2 * x)


@torch.no_grad()
def mouth_truth(sd, feats, opt, device="cpu") -> torch.Tensor:
    """Float64 ``generate_sequences`` output [n/2, out] on ``device``: the appended rows, the pairing, exact eval-mode
    BatchNorm, the LSTM equations and the kept rows."""
    p = lambda k: _t64(sd[k], device)      # noqa: E731
    x = _t64(np.asarray(feats, np.float32), device)
    n, D = x.shape
    ff = opt.frame_future
    if ff:
        x = torch.cat([x, x[-1:].expand(2 * ff, D)])
    x = x.reshape(-1, 2 * D)

    def lin(v, name):
        return v @ p(name + ".weight").T + p(name + ".bias")

    def bn(v, name):
        return (v - p(name + ".running_mean")) / torch.sqrt(p(name + ".running_var") + BN_EPS) * p(name + ".weight") + p(name + ".bias")
    y = lin(_lrelu(bn(lin(x, "downsample.0"), "downsample.1")), "downsample.3")
    for k in range(3):
        y = lstm_layer_truth(y, p(f"LSTM.weight_ih_l{k}"), p(f"LSTM.weight_hh_l{k}"), p(f"LSTM.bias_ih_l{k}"),
                             p(f"LSTM.bias_hh_l{k}"))
    y = y[ff:]
    y = _lrelu(bn(lin(y, "fc.0"), "fc.1"))
    y = _lrelu(bn(lin(y, "fc.3"), "fc.4"))
    return lin(y, "fc.6")


# ------------------------------------------------------------------------------------------------------------------
# Emulator of the kernels, on the packed arrays
# ------------------------------------------------------------------------------------------------------------------
def _rnn_emulate(x, w_ih, b, w_hh, b_hn, G: int, H: int, cl: int):
    """The recurrence of csrc/lspr.cu in float64: x [T, In]; packed row u*G + g; CTA c owns the row block
    [c G H / cl, (c+1) G H / cl) of w_hh and the units [c H / cl, (c+1) H / cl)."""
    T = x.shape[0]
    U = H // cl
    xproj = (x @ w_ih.reshape(G * H, -1).T + b).reshape(T, H, G)
    w_hh = w_hh.reshape(cl, G * U, H)
    h = np.zeros(H)
    c = np.zeros(H)
    out = np.empty((T, H))
    for t in range(T):
        gh = np.concatenate([w_hh[k] @ h for k in range(cl)]).reshape(H, G)       # every CTA from its own copy of h
        xg = xproj[t]
        if G == 3:
            r = 1 / (1 + np.exp(-(xg[:, 0] + gh[:, 0])))
            z = 1 / (1 + np.exp(-(xg[:, 1] + gh[:, 1])))
            n = np.tanh(xg[:, 2] + r * (gh[:, 2] + b_hn))
            h = n + z * (h - n)
        else:
            i = 1 / (1 + np.exp(-(xg[:, 0] + gh[:, 0])))
            f = 1 / (1 + np.exp(-(xg[:, 1] + gh[:, 1])))
            g = np.tanh(xg[:, 2] + gh[:, 2])
            o = 1 / (1 + np.exp(-(xg[:, 3] + gh[:, 3])))
            c = f * c + i * g
            h = o * np.tanh(c)
        out[t] = h
    return out


def emulate_apc(packed, mel, layers: int, residual: bool = False, cl: int = 16, hidden: int = 512) -> np.ndarray:
    """``packed(which)`` returns lspr_debug_packed's array ``which`` of an APC handle."""
    x = np.asarray(mel, np.float32).astype(np.float64)
    for l in range(layers):
        a = [packed(4 * l + j).astype(np.float64) for j in range(4)]
        y = _rnn_emulate(x, a[0], a[1], a[2], a[3], 3, hidden, cl)
        if residual and l + 1 < layers and x.shape[1] == hidden:
            y = y + x
        x = y
    return x


def emulate_mouth(packed, feats, frame_future: int, cl: int = 8) -> np.ndarray:
    """``packed(which)`` returns lspr_debug_packed's array ``which`` of a MOUTH handle."""
    x = np.asarray(feats, np.float32).astype(np.float64)
    n, D = x.shape
    steps = n // 2 + frame_future

    def stage(v, s, leaky):
        w, sc, sh = (packed(12 + 3 * s + j).astype(np.float64) for j in range(3))
        y = (v @ w.reshape(sc.shape[0], -1).T) * sc + sh
        return np.where(y > 0, y, 0.2 * y) if leaky else y
    src = np.minimum(np.arange(2 * steps), n - 1)                # the appended rows are the last row, by clamping
    y = stage(x[src].reshape(steps, 2 * D), 0, True)
    y = stage(y, 1, False)
    for k in range(3):
        a = [packed(4 * k + j).astype(np.float64) for j in range(4)]
        y = _rnn_emulate(y, a[0], a[1], a[2], None, 4, LSTM_H, cl)
    y = y[frame_future:]
    y = stage(y, 2, True)
    y = stage(y, 3, True)
    return stage(y, 4, False)


def exact_fold(sd):
    """A copy of ``sd`` on which every fold lspr_load_weights does is exact in fp32, so the packed arrays hold the
    float64 model exactly and the emulator can be held to float64 accuracy against the truth: recurrent biases on a
    2^-16 grid (b_ih + b_hh needs no rounding), BatchNorm mean and bias on a 2^-12 grid, running_var = 2^30 (so
    running_var + 1e-5f is 2^30 in fp32, its sqrt 2^15, and the float64 sqrt(running_var + 1e-5) is 2^15 to 5e-15
    relative) and weight = 2^15 times a value on a 2^-8 grid, which makes the folded scale that value exactly.  How the
    fold rounds on general weights is pinned separately (``fold_bn_fp32``)."""
    q = lambda v, step: torch.round(v / step) * step       # noqa: E731
    out = OrderedDict()
    for k, v in sd.items():
        v = v.detach().clone()
        if "bias_ih" in k or "bias_hh" in k:
            v = q(v, 2.0 ** -16)
        elif k.startswith(("downsample.1.", "fc.1.", "fc.4.")):
            if k.endswith(".weight"):
                v = q(v, 2.0 ** -8) * 2.0 ** 15
            elif k.endswith((".bias", ".running_mean")):
                v = q(v, 2.0 ** -12)
            elif k.endswith(".running_var"):
                v = torch.full_like(v, 2.0 ** 30)
        elif k.endswith(".bias") and k.startswith(("downsample.0", "fc.0", "fc.3")):
            v = q(v, 2.0 ** -12)
        out[k] = v
    return out


def fold_bn_fp32(sd, lin: str, bn: str):
    """The scale / shift lspr_load_weights folds, restated in fp32 (numpy rounds each operation as the host code does)."""
    f = lambda k: sd[k].numpy().astype(np.float32)      # noqa: E731
    s = f(bn + ".weight") / np.sqrt(f(bn + ".running_var") + np.float32(BN_EPS))
    return s, (f(lin + ".bias") - f(bn + ".running_mean")) * s + f(bn + ".bias")
