"""GPU *library* baseline (not a product path): the oracle restatement executed by PyTorch eager + cuDNN on the
same H100 - what the unmodified reference module would run (base_model.py:46-47 sets cudnn.benchmark) - in
fp32, TF32 and bf16-autocast/channels_last.  Prints frames/s so the hand-written kernels can be put beside it."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from oracle import f2f_oracle as O  # noqa: E402


def timed(fn, n=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def main():
    variant = sys.argv[1] if len(sys.argv) > 1 else "large"
    batch = int(sys.argv[2]) if len(sys.argv) > 2 else 8
    torch.backends.cudnn.benchmark = True
    sd = {k: v.cuda() for k, v in O.make_state_dict(variant, "A").items()}
    fm, cand = O.make_inputs(batch, 512, 512)
    x = torch.cat([fm, cand], 1).cuda()
    ref = O.generator_forward({k: v.cpu() for k, v in sd.items()}, x[:1].cpu(), variant)
    res = {}
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    ms = timed(lambda: O.generator_forward(sd, x, variant))
    err = (O.generator_forward(sd, x[:1], variant).cpu() - ref).abs().max().item()
    res["fp32"] = (batch / ms * 1e3, err)
    torch.backends.cudnn.allow_tf32 = True
    ms = timed(lambda: O.generator_forward(sd, x, variant))
    err = (O.generator_forward(sd, x[:1], variant).cpu() - ref).abs().max().item()
    res["tf32"] = (batch / ms * 1e3, err)
    xc = x.contiguous(memory_format=torch.channels_last)
    sdc = {k: (v.contiguous(memory_format=torch.channels_last) if v.dim() == 4 else v) for k, v in sd.items()}

    def bf16():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            return O.generator_forward(sdc, xc, variant)
    ms = timed(bf16)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        err = (O.generator_forward(sdc, xc[:1], variant).float().cpu() - ref).abs().max().item()
    res["bf16_autocast_channels_last"] = (batch / ms * 1e3, err)
    for k, (fps, err) in res.items():
        print(f"cudnn-eager {variant} B{batch} 512x512 {k}: {fps:.1f} frames/s, max|out-oracle(cpu fp32)| {err:.3g}", flush=True)


if __name__ == "__main__":
    main()
