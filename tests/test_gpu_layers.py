"""Every conv launch of one forward against the float64 reference of its own layer (tests/layer_reference.py), in both
precision modes, on the configurations that together reach every kernel variant the planner can select
(tests/test_layer_reference.py::test_gpu_configs_cover_every_planner_variant keeps that list honest).

Each layer is checked on exactly the activations it consumed (read back from the device), at every output pixel and
channel, against a per-element bound derived from the kernel's arithmetic, so an error cannot carry over from an
earlier layer and a wrong tile, tap, limb or channel block shows up at the layer that made it.
"""
from __future__ import annotations

import ctypes as C
import os
import sys
import types

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import layer_reference as R  # noqa: E402
from oracle import f2f_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

# (variant, recipe, batch, height, width)
GPU_LAYER_CONFIGS = [
    ("normal", "B", 1, 256, 256),      # patch tail CL 1; patch BN 64 with and without split-K; umma 64/128 split-K
    ("normal", "B", 8, 512, 512),      # patch BN 128 / 64 / tail at CL 2; umma 64 and 128 without split
    ("large", "A", 33, 512, 256),      # patch BN 128 CL 1 (odd M-tile counts, odd batch); several images per umma tile
]


def variant_key(info, g) -> tuple:
    return ("patch" if g.kernel == 1 else "umma", g.bn, info.kind == R.KIND_TAIL, g.cluster, g.n_split > 1)


def _host_variants(variant, batch, hh, ww):
    from livespeechportraits_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    _lib.check(lib.lspg_create(C.byref(h), _lib.LSPG_VARIANT[variant], 64, 8, 13, 3, -1))
    try:
        return set(R.planner_variants(lib, h, batch, hh, ww))
    finally:
        lib.lspg_destroy(h)


def _ulp_f16(hi: torch.Tensor) -> torch.Tensor:
    a = hi.float().abs()
    _, e = torch.frexp(a)                                  # a = m * 2^e, m in [0.5, 1)
    ulp = torch.ldexp(torch.ones_like(a), (e - 11).clamp(min=-24))
    return torch.where(a == 0, torch.full_like(a, 2.0 ** -24), ulp)


def _run_config(variant, recipe, batch, hh, ww, mode):
    from livespeechportraits_b200 import _lib
    from livespeechportraits_b200.generator import Feature2Face_G
    opt = types.SimpleNamespace(isTrain=False, size=variant, n_downsample_G=8, ngf=64, fp16=0)
    sd = O.make_state_dict(variant, recipe)
    net = Feature2Face_G(opt, precision=mode)
    net.load_state_dict(sd, strict=True)
    net = net.cuda().eval()
    fm, cand = O.make_inputs(batch, hh, ww)
    x = torch.cat([fm, cand], 1)
    out = net(x.cuda())
    torch.cuda.synchronize()
    lib, h = net._lib, net._handle
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    dev = torch.device("cuda")

    def act(tid):
        if mode == "parity":
            hi = net.debug_read_tensor(tid, batch, hh, ww, 0)
            lo = net.debug_read_tensor(tid, batch, hh, ww, 1)
            assert torch.isfinite(hi).all() and torch.isfinite(lo).all(), f"tensor {tid}: non-finite limb"
            bad = lo.float().abs() > _ulp_f16(hi) / 2
            assert not bad.any(), f"tensor {tid}: |lo| > ulp(hi)/2 at {bad.nonzero()[0].tolist()}"
            return [hi.to(dev).double(), lo.to(dev).double()]
        t = net.debug_read_tensor(tid, batch, hh, ww, 0)
        assert torch.isfinite(t).all(), f"tensor {tid}: non-finite"
        return [t.to(dev).double()]

    # input packer, bit-exact
    s2d = R.pack_s2d(x)
    if mode == "parity":
        hi = net.debug_read_tensor(0, batch, hh, ww, 0)
        lo = net.debug_read_tensor(0, batch, hh, ww, 1)
        ehi = s2d.half()
        assert torch.equal(hi.view(torch.int16), ehi.view(torch.int16)), "packer: limb 0 != fp16(x)"
        assert torch.equal(lo.view(torch.int16), (s2d - ehi.float()).half().view(torch.int16)), "packer: limb 1 != fp16(x - hi)"
    else:
        t0 = net.debug_read_tensor(0, batch, hh, ww, 0)
        assert torch.equal(t0.view(torch.int16), s2d.bfloat16().view(torch.int16)), "packer: tensor 0 != bf16(x)"
    tensors = {0: act(0)}
    for q in range(4):
        assert all((t[..., q * 16 + 13:q * 16 + 16] == 0).all() for t in tensors[0]), "space-to-depth pad channels must be zero"

    nl = C.c_int()
    _lib.check(lib.lspg_num_layers(h, C.byref(nl)))
    worst = {}                                        # (variant key, tier) -> (err/bound, layer, conv key)
    failures = []
    for i in range(nl.value):
        info = _lib.LspgLayerInfo()
        _lib.check(lib.lspg_layer_info_get(h, i, C.byref(info)))
        g = _lib.LspgLayerGeo()
        _lib.check(lib.lspg_debug_layer_geo(h, i, batch, hh, ww, C.byref(g)))
        key = variant_key(info, g)
        for tid in [info.src[s] for s in range(info.n_src)] + ([info.res] if info.res >= 0 else []):
            if tid not in tensors:
                tensors[tid] = act(tid)
        xin = [torch.cat([tensors[info.src[s]][li] for s in range(info.n_src)], dim=3) for li in range(len(tensors[0]))]
        res = tensors[info.res] if info.res >= 0 else None
        spec = R.layer_spec(sd, info, mode, dev)
        sem_v, sem_b, ker_v, ker_b = R.layer_full(spec, xin, mode, g, res)
        if info.kind == R.KIND_TAIL:
            got = out.double().permute(0, 2, 3, 1)
        else:
            tensors[info.out] = act(info.out)
            got = sum(tensors[info.out])
        for tier, val, bnd in (("semantic", sem_v, sem_b), ("kernel", ker_v, ker_b)):
            ratio = (got - val).abs() / bnd
            r = ratio.max().item()
            if r > worst.get((key, tier), (-1.0,))[0]:
                worst[(key, tier)] = (r, i, info.conv_key.decode())
            if not r <= 1.0:
                n, y, xq, c = (int(v) for v in np.unravel_index(int(ratio.argmax()), tuple(ratio.shape)))
                failures.append(f"{variant}/{recipe} B{batch} {hh}x{ww} {mode}: layer {i} {info.conv_key.decode()} variant {key} "
                                f"{tier} bound: err/bound {r:.3g} at (n={n}, y={y}, x={xq}, c={c}) "
                                f"got {got[n, y, xq, c].item():.9g} ref {val[n, y, xq, c].item():.9g} "
                                f"bound {bnd[n, y, xq, c].item():.3g}; " + _where(info, g, xin[0].shape, n, y, xq, c, sms))
        del sem_v, sem_b, ker_v, ker_b
        for tid in list(tensors):                     # keep only what later layers read
            if tid != 0 and tid not in _later_reads(lib, h, i, nl.value):
                del tensors[tid]
    # fused tensor2im of the same run
    img = net.render_image(x.cuda(), None).cpu().numpy()
    assert np.array_equal(img, O.tensor2im(out.cpu())), "render_image != tensor2im(render)"
    return worst, sms, failures


def _where(info, g, src_shape, n, y, x, c, sms) -> str:
    """Tile, GEMM column and CTA / local tile of output element (n, y, x, c).  Tiles count x fastest, then y, then image
    group, then N tile, then phase (the folded upsample's four phases are separate GEMMs); the tail is one GEMM whose 16
    columns are (phase, channel), so its output pixel (y, x) is source pixel (y/2, x/2), column (y%2*2 + x%2)*3 + c."""
    up = info.kind in (R.KIND_UP, R.KIND_TAIL)
    ys, xs = (y // 2, x // 2) if up else (y, x)
    ph = (y % 2) * 2 + x % 2
    z, col = (ph, c) if info.kind == R.KIND_UP else ((0, ph * 3 + c) if info.kind == R.KIND_TAIL else (0, c))
    sub = 2 if info.kind == R.KIND_S2 else 1
    tiles_x, tiles_y = src_shape[2] // sub // g.tile_w, src_shape[1] // sub // g.tile_h
    mt = xs // g.tile_w + tiles_x * (ys // g.tile_h + tiles_y * (n // g.tile_n))
    t = mt + g.m_tiles * (col // g.bn + g.n_tiles * z)
    ctas = min(g.ctas, sms)
    return (f"tile {t} (GEMM column {col}, phase {z}, row {((n % g.tile_n) * g.tile_h + ys % g.tile_h) * g.tile_w + xs % g.tile_w}; CTA {t % ctas}, local tile "
            f"{t // ctas}, {'odd' if (t // ctas) % 2 else 'even'}{', split 0' if g.n_split > 1 else ''})")


def _later_reads(lib, h, i, n):
    from livespeechportraits_b200 import _lib
    ids = set()
    for j in range(i + 1, n):
        info = _lib.LspgLayerInfo()
        lib.lspg_layer_info_get(h, j, C.byref(info))
        ids.update(info.src[s] for s in range(info.n_src))
        if info.res >= 0:
            ids.add(info.res)
    return ids


@pytest.mark.parametrize("mode", ["parity", "fast"])
@pytest.mark.parametrize("cfg", GPU_LAYER_CONFIGS, ids=lambda c: f"{c[0]}{c[1]}_b{c[2]}_{c[3]}x{c[4]}")
def test_every_layer_against_float64_reference(cfg, mode):
    worst, sms, failures = _run_config(*cfg, mode)
    for key, tier in sorted(worst):
        r, i, k = worst[(key, tier)]
        print(f"[layers] {cfg} {mode} {key} {tier}: worst err/bound {r:.3g} (layer {i} {k})")
    missed = _host_variants(*[cfg[0]] + list(cfg[2:])) - {key for key, _ in worst}
    if missed:
        print(f"[layers] device has {sms} SMs: variants this config reaches at 132 SMs that did not run: {sorted(missed)}")
    assert not failures, "\n".join(failures[:8])
