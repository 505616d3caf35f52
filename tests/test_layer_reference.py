"""Host checks of the per-layer float64 reference and its error bound (tests/layer_reference.py), and of the list of
configurations the GPU per-layer test runs (tests/test_gpu_layers.py).

* The reference is right: chained over the network it reproduces the float64 oracle.
* The bound is right and has teeth: a float64 emulation of the kernels' arithmetic (operand limbs, fp32 accumulator
  rounded after every k16 MMA in the kernel's K order, split-K partials, fp32 epilogue, 16-bit stores) passes it at
  every layer, and six small defects of that arithmetic each fail it at some layer.
* The GPU configurations reach every kernel variant the planner can select.
"""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import layer_reference as R  # noqa: E402
from oracle import f2f_oracle as O  # noqa: E402
from livespeechportraits_b200 import _lib  # noqa: E402

CPU_CONFIGS = [("normal", "B"), ("large", "A")]       # at 256 x 256, one frame
HW = 256


class Net:
    """Host-only handle: layer rows and the planner's geometry at 132 SMs."""

    def __init__(self, variant, sd=None):
        self.lib = _lib.load()
        self.h = C.c_void_p()
        _lib.check(self.lib.lspg_create(C.byref(self.h), _lib.LSPG_VARIANT[variant], 64, 8, 13, 3, -1))
        n = C.c_int()
        _lib.check(self.lib.lspg_num_layers(self.h, C.byref(n)))
        self.layers = []
        for i in range(n.value):
            info = _lib.LspgLayerInfo()
            _lib.check(self.lib.lspg_layer_info_get(self.h, i, C.byref(info)))
            self.layers.append(info)
        if sd is not None:
            keep = [(k.encode(), v.float().contiguous()) for k, v in sd.items() if not k.endswith("num_batches_tracked")]
            arr = (_lib.LspgTensor * len(keep))()
            for i, (k, t) in enumerate(keep):
                arr[i].name, arr[i].numel, arr[i].data = k, t.numel(), C.cast(t.data_ptr(), C.POINTER(C.c_float))
            _lib.check(self.lib.lspg_load_weights(self.h, arr, len(keep)))

    def geo(self, i, b, hh, ww):
        g = _lib.LspgLayerGeo()
        _lib.check(self.lib.lspg_debug_layer_geo(self.h, i, b, hh, ww, C.byref(g)))
        return g

    def close(self):
        self.lib.lspg_destroy(self.h)


def _store(v: torch.Tensor, mode: str):
    """What the epilogue stores for fp32 value v: PARITY (hi, lo) fp16 limbs, FAST bf16."""
    y = v.float()
    if mode == "parity":
        hi = y.half()
        return hi.double(), (y - hi.float()).half().double()
    return (y.bfloat16().double(),)


def _chain(sd, net, x, mode):
    """Per-layer reference chained over the network.  mode None: float64 all through (no stores);
    otherwise each layer reads the stored form of the previous reference outputs.  Returns (tensors, tail NCHW)."""
    s = R.pack_s2d(x.double())
    tensors = {0: _store(s, mode) if mode else (s,)}
    tail = None
    for i, info in enumerate(net.layers):
        spec = R.layer_spec(sd, info, mode or "parity")
        xin = torch.cat([sum(tensors[info.src[j]]) for j in range(info.n_src)], dim=3)
        res = [sum(tensors[info.res])] if info.res >= 0 else None
        g = net.geo(i, x.shape[0], x.shape[2], x.shape[3])
        val = R.layer_full(spec, [xin], mode or "parity", g, res, value_only=True)
        if info.kind == R.KIND_TAIL:
            tail = val.permute(0, 3, 1, 2)
        else:
            tensors[info.out] = _store(val, mode) if mode else (val,)
    return tensors, tail


@pytest.fixture(scope="module", params=CPU_CONFIGS, ids=lambda c: f"{c[0]}{c[1]}")
def chained(request):
    variant, recipe = request.param
    sd = O.make_state_dict(variant, recipe)
    net = Net(variant, sd)
    fm, cand = O.make_inputs(1, HW, HW)
    x = torch.cat([fm, cand], 1)
    yield variant, recipe, sd, net, x
    net.close()


def test_reference_chain_matches_float64_oracle(chained):
    """Chaining the per-layer reference reproduces the oracle (pinned bit-exact against the reference module) run on a
    float64 copy of the state dict, to float64 rounding."""
    variant, _, sd, net, x = chained
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    want = O.generator_forward(sd64, x.double(), variant)
    _, got = _chain(sd, net, x, None)
    err = (got - want).abs().max().item()
    assert err < 1e-12, err


def test_fast_weights_match_packed(chained):
    """The bf16 weights the FAST reference multiplies, built from the state dict, equal what the library packed (limb 2),
    so a packing error reports here and not as a kernel error."""
    _, _, sd, net, _ = chained
    for i, info in enumerate(net.layers):
        spec = R.layer_spec(sd, info, "fast")
        count = info.n_phases * info.cout_pad * info.k_total
        buf = np.zeros(count, np.uint16)
        _lib.check(net.lib.lspg_layer_packed(net.h, i, 2, buf.ctypes.data, count))
        packed = torch.from_numpy((buf.astype(np.uint32) << 16).view(np.float32).copy()).double()
        packed = packed.view(info.n_phases, info.cout_pad, -1, spec.cin)          # [phase][cout][tap][channel]
        for z in range(len(spec.phases)):
            for t, off in enumerate(spec.offsets[z]):
                if info.kind == R.KIND_TAIL:          # one GEMM: columns (phase, channel), taps (dy, dx) in {-1,0,1}^2
                    got = packed[0, z * spec.cout:(z + 1) * spec.cout, (off[0] + 1) * 3 + off[1] + 1].t()
                else:
                    got = packed[z, :spec.cout, t].t()
                assert torch.equal(got, spec.w[z][off]), (i, info.conv_key, z, off)


def _tile_pixels(g, t, batch, hs, ws):
    tiles_x, tiles_y = ws // g.tile_w, hs // g.tile_h
    mt = t % g.m_tiles
    tx, ty, tn = mt % tiles_x, (mt // tiles_x) % tiles_y, mt // (tiles_x * tiles_y)
    r = torch.arange(128)
    x = tx * g.tile_w + r % g.tile_w
    y = ty * g.tile_h + (r // g.tile_w) % g.tile_h
    n = tn * g.tile_n + r // (g.tile_w * g.tile_h)
    keep = n < batch
    return n[keep], y[keep], x[keep]


def sample_pixels(g, batch, hs, ws, seed):
    """Deterministic sample of source-grid pixels: every pixel at 32 x 32 and below; otherwise all rows of the first and the
    last tile, of local tiles 0 and 1 of CTA 0 (one per consumer warpgroup), of the tiles at the four corners (TMA's zero
    fill is the padding there), every row of the last image's first tile, and random pixels."""
    if hs * ws <= 32 * 32:
        return R.grid_pixels(batch, hs, ws)
    tiles_x, tiles_y = ws // g.tile_w, hs // g.tile_h
    corner = [0, tiles_x - 1, tiles_x * (tiles_y - 1), tiles_x * tiles_y - 1]
    last_img = (batch - 1) // g.tile_n * tiles_x * tiles_y
    parts = [_tile_pixels(g, t, batch, hs, ws) for t in {0, g.m_tiles - 1, g.ctas % g.m_tiles, last_img, *corner}]
    rng = np.random.Generator(np.random.PCG64(seed))
    k = 96
    parts.append((torch.from_numpy(rng.integers(0, batch, k)), torch.from_numpy(rng.integers(0, hs, k)),
                  torch.from_numpy(rng.integers(0, ws, k))))
    n, y, x = (torch.cat([p[j] for p in parts]) for j in range(3))
    key = torch.unique((n * hs + y) * ws + x)
    return key // (hs * ws), (key // ws) % hs, key % ws


MUTATIONS = ["none", "drop_hi_lo", "drop_lo_hi", "drop_res_lo", "shift_tap", "swap_channel_groups", "zero_last_tap"]
EVERY_LAYER = ("drop_hi_lo", "drop_lo_hi")          # must fail the kernel-arithmetic bound at every layer


def fast_short_tap(info, g):
    """Kernel tap index of the last tap of a short tap group, or None.  In FAST, conv_patch_kernel without a cluster fetches
    the weights of several taps with one TMA box (the planner reports its taps in w_box_taps), and a last group with fewer
    taps than the box is completed by TMA's zero fill."""
    tps = g.w_box_taps[_lib.LSPG_MODE["fast"]]
    return info.n_taps - 1 if info.n_taps % tps else None


def emulate(spec, ins, n, y, x, z, mode, g, res, mutation, short_tap=None):
    """The kernel's arithmetic at source-grid pixels (n, y, x) of phase z, in float64 with explicit roundings: the limb
    products of each k16 MMA are summed and the accumulator is rounded to fp32, in the kernel's K order; split-K partials
    are summed in fp32; the epilogue rounds to fp32 after the fma and after each residual limb; the store rounds to the
    16-bit format.  ins: stored limbs of the concatenated sources; res: stored limbs of the residual at the output pixels."""
    p = n.shape[0]
    total = torch.zeros(p, spec.cout, dtype=torch.float64)
    first_off = spec.offsets[z][0]
    prods = [q for q in R.LIMB_PRODUCTS[mode]
             if not (mutation == "drop_hi_lo" and q == (0, 1)) and not (mutation == "drop_lo_hi" and q == (1, 0))]
    items = R.k_items(spec, z, g.kernel == 1)
    for s in range(g.n_split):
        acc = torch.zeros(p, spec.cout, dtype=torch.float64)
        for item in items[s * g.split_len:(s + 1) * g.split_len]:
            for off, ch in item:
                if mutation == "zero_last_tap" and spec.offsets[z].index(off) == short_tap:
                    continue
                dx = off[1] + 1 if (mutation == "shift_tap" and off == first_off) else off[1]
                a = [R.gather(t, n, y, x, spec.stride, off[0], dx, ch) for t in ins]
                w = R.kernel_weights(spec, z, off, ch, mode)
                for k in range(0, a[0].shape[1], 16):
                    for ia, iw in prods:
                        acc = (acc + a[ia][:, k:k + 16] @ w[iw][k:k + 16]).float().double()
        total = (total + acc).float().double() if g.n_split > 1 else acc
    v = (total * R.kernel_scale(spec, mode) + spec.shift32.double()).float().double()
    if spec.kind == R.KIND_TAIL:
        return torch.tanh(v.float()).double()
    if res is not None:
        for li, r in enumerate(res):
            if not (mutation == "drop_res_lo" and li == 1):
                v = (v + r).float().double()
    if spec.relu:
        v = torch.relu(v)
    if mutation == "swap_channel_groups":
        v = torch.cat([v[:, 4:8], v[:, 0:4], v[:, 8:]], 1)
    return sum(_store(v, mode))


@pytest.mark.parametrize("mode", ["parity", "fast"])
def test_emulated_kernel_passes_bound_and_mutations_fail(chained, mode):
    """The emulated kernel stays within half of the semantic bound and within the kernel-arithmetic bound at every layer.  Each mutation of its arithmetic exceeds the
    kernel-arithmetic bound: a dropped limb product at every layer, the others at some layer.  The FAST short-tap-group
    mutation applies only to launches that have a short group."""
    variant, recipe, sd, net, x = chained
    tensors, _ = _chain(sd, net, x, mode)
    b = x.shape[0]
    mutations = [m for m in MUTATIONS if not (mode == "fast" and m in ("drop_hi_lo", "drop_lo_hi", "drop_res_lo"))
                 and not (mode == "parity" and m == "zero_last_tap")]
    caught = {m: [] for m in mutations if m != "none"}
    missed = {m: [] for m in mutations if m in EVERY_LAYER}
    weakest = {m: (float("inf"), -1) for m in missed}
    worst = [0.0, 0.0]
    for i, info in enumerate(net.layers):
        spec = R.layer_spec(sd, info, mode)
        g = net.geo(i, b, HW, HW)
        short = fast_short_tap(info, g) if mode == "fast" else None
        ins = [torch.cat([tensors[info.src[j]][li] for j in range(info.n_src)], dim=3) for li in range(len(tensors[0]))]
        hs, ws = (ins[0].shape[1] // 2, ins[0].shape[2] // 2) if info.kind == R.KIND_S2 else ins[0].shape[1:3]
        n, y, xx = sample_pixels(g, b, hs, ws, seed=i)
        layer_ratio = {m: 0.0 for m in missed}
        for z in range(len(spec.phases)):
            oy, ox = R.output_pixels(spec, z, y, xx)
            res = [t[n, oy, ox] for t in tensors[info.res]] if info.res >= 0 else None
            sem, ker = R.evaluate(spec, ins, n, y, xx, z, mode, g, res)
            for m in mutations:
                if m not in EVERY_LAYER and m != "none" and caught[m]:
                    continue
                if m == "zero_last_tap" and short is None:
                    continue
                got = emulate(spec, ins, n, y, xx, z, mode, g, res, m, short)
                ratio = ((got - ker.value).abs() / ker.bound).max().item()
                if m == "none":
                    rs = ((got - sem.value).abs() / sem.bound).max().item()
                    worst = [max(worst[0], rs), max(worst[1], ratio)]
                    # the kernel-arithmetic bound is mostly the 16-bit store's rounding, which a round-to-nearest store
                    # can nearly reach, so only the semantic bound is held to a margin
                    assert rs <= 0.5 and ratio <= 1.0, \
                        f"layer {i} {info.conv_key.decode()} phase {z}: emulated kernel at {rs:.3g} / {ratio:.3g} of the bounds"
                    continue
                if m in layer_ratio:
                    layer_ratio[m] = max(layer_ratio[m], ratio)
                if ratio > 1.0:
                    caught[m].append(i)
        for m, r in layer_ratio.items():
            weakest[m] = min(weakest[m], (r, i))
            if r <= 1.0:
                missed[m].append(i)
    print(f"[bound] {variant}/{recipe} {mode}: emulated kernel reaches {worst[0]:.3g} of the semantic bound and {worst[1]:.3g} "
          f"of the kernel-arithmetic bound; first layer catching each mutation { {m: v[:1] for m, v in caught.items()} }; "
          f"weakest layer for the dropped limb products (err/bound, layer) {weakest}")
    assert all(caught.values()), f"mutations the bound does not catch: {[m for m, v in caught.items() if not v]}"
    assert not any(missed.values()), f"layers where a dropped limb product stays within the bound: {missed}"


# (variant, batch, H, W) swept for the coverage check: powers of two from 256 to 2048, batch 1-129
SWEEP_SHAPES = [(hh, ww) for hh in (256, 512, 1024, 2048) for ww in (256, 512, 1024, 2048) if hh * ww <= 1024 * 1024]
SWEEP_BATCHES = list(range(1, 40)) + [48, 63, 64, 65, 96, 127, 128, 129]


def test_gpu_configs_cover_every_planner_variant():
    """Every (kernel, BN, tail, cluster, split-K) the planner selects for some accepted shape at 132 SMs is run by a
    configuration of the GPU per-layer test; a planner change that makes a new variant reachable fails here until a
    configuration for it is added."""
    from test_gpu_layers import GPU_LAYER_CONFIGS
    reachable, covered = {}, set()
    for variant in ("normal", "large"):
        net = Net(variant)
        for hh, ww in SWEEP_SHAPES:
            for b in SWEEP_BATCHES:
                for key in R.planner_variants(net.lib, net.h, b, hh, ww):
                    reachable.setdefault(key, (variant, b, hh, ww))
        for v, _, b, hh, ww in GPU_LAYER_CONFIGS:
            if v == variant:
                covered |= set(R.planner_variants(net.lib, net.h, b, hh, ww))
        net.close()
    missing = {k: reachable[k] for k in reachable if k not in covered}
    assert not missing, f"variants no GPU layer config runs (key: first shape that selects it): {missing}"
