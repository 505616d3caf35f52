"""Time the recurrent audio networks (include/lspr.h) on the GPU against the reference modules on cuDNN.

    python tests/gpu_scripts/rnn_bench.py [--iters 10]

Prints ONE JSON line.  At T = 1374 mel frames (the shipped clip) and T = 72000 (10 minutes):
  * the library: kernel time per call from torch.profiler (the recurrence kernels rnn_layer_kernel and the GEMMs
    gemm_nt_kernel, summed, mean over --iters calls), the recurrence's time per step and layer, and the CUDA-event time of
    ApcEncoder.forward / MouthGenerator.generate on device-resident input (Audio2Mouth on T APC rows: T/2 frames);
  * the reference modules (torch.nn.GRU stack as APC_encoder runs it, the Audio2Feature LSTM path) on cuDNN on the same
    card, CUDA-event time, with torch.backends.cudnn.allow_tf32 True and False, each with its max-abs error against the
    float64 truth (T = 1374 only: the float64 truth of the 10-minute clip is not recomputed here);
  * the library's own max-abs error against the float64 truth at T = 1374.
Card name and power limit come from a read-only nvidia-smi query in the same run.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from lle_bench import card, event_ms  # noqa: E402
from livespeechportraits_b200.recurrent import ApcEncoder, MouthGenerator  # noqa: E402
from oracle import rnn_oracle as R  # noqa: E402


def kernel_ms(fn, iters):
    """Mean per call of (recurrence kernels, GEMM kernels) from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    rec = gemm = 0.0
    for ev in prof.events():
        t = getattr(ev, "device_time", None)
        t = (t if t is not None else getattr(ev, "cuda_time", 0.0)) / 1000.0
        if "rnn_layer_kernel" in ev.name:
            rec += t
        elif "gemm_nt_kernel" in ev.name:
            gemm += t
    return rec / iters, gemm / iters


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    name, limit = card()
    res = {"card": name, "power_limit": limit, "cases": {}}
    asd = R.make_apc_state_dict("A", 0)
    mopt = R.default_mouth_opt()
    msd = R.make_mouth_state_dict(mopt, "A", 0)
    enc = ApcEncoder(asd, device=dev)
    mouth = MouthGenerator(mopt, msd, device=dev)
    apc_ref = R.apc_module(asd).to(dev).eval()
    mouth_ref = R.mouth_module(mopt, msd).to(dev).eval()

    def apc_cudnn(x):
        with torch.no_grad():
            y = x[None]
            for rnn in apc_ref.rnns:
                y = rnn(y)[0]
            return y[0]

    def mouth_cudnn(f):
        ff = mopt.frame_future
        with torch.no_grad():
            x = torch.cat([f, f[-1:].expand(2 * ff, f.shape[1])])[None]
            return mouth_ref(x)[0, ff:]

    for T in (1374, 72000):
        mel = torch.from_numpy(R.make_mel(T, seed=T)).to(dev)
        feats = torch.from_numpy(R.make_feats(T, seed=T)).to(dev)
        r = {}
        for label, fn, steps, layers in (("apc", lambda: enc.forward(mel), T, 3),
                                         ("mouth", lambda: mouth.generate(feats), T // 2 + mopt.frame_future, 3)):
            for _ in range(2):
                fn()
            torch.cuda.synchronize()
            iters = a.iters if T < 10000 else max(2, a.iters // 5)
            rec, gemm = kernel_ms(fn, iters)
            r[label] = {"steps_per_layer": steps, "recurrence_kernel_ms": round(rec, 3), "gemm_kernel_ms": round(gemm, 3),
                        "us_per_step_per_layer": round(rec * 1e3 / (steps * layers), 3),
                        "call_ms": round(event_ms(fn, iters), 3)}
        if T == 1374:
            at = R.apc_truth(asd, mel.cpu().numpy()).numpy()
            mt = R.mouth_truth(msd, feats.cpu().numpy(), mopt).numpy()
            r["apc"]["max_abs_err_vs_f64"] = float(np.abs(enc.forward(mel).cpu().numpy() - at).max())
            r["mouth"]["max_abs_err_vs_f64"] = float(np.abs(mouth.generate(feats).cpu().numpy() - mt).max())
        for tf32 in (True, False):
            torch.backends.cudnn.allow_tf32 = tf32
            for label, fn in (("apc", lambda: apc_cudnn(mel)), ("mouth", lambda: mouth_cudnn(feats))):
                key = f"cudnn_{label}_allow_tf32_{tf32}"
                try:
                    for _ in range(2):
                        fn()
                    torch.cuda.synchronize()
                except RuntimeError as exc:          # cuDNN refuses some shapes; report it instead of a time
                    r[key] = {"error": str(exc).splitlines()[0]}
                    continue
                r[key] = {"call_ms": round(event_ms(fn, a.iters if T < 10000 else 2), 3)}
                if T == 1374:
                    truth = at if label == "apc" else mt
                    r[key]["max_abs_err_vs_f64"] = float(np.abs(fn().cpu().numpy() - truth).max())
        torch.backends.cudnn.allow_tf32 = True
        res["cases"][str(T)] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
