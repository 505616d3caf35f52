"""Float64 reference of one conv launch of the generator, and the per-element error bound its CUDA kernel must meet.

The layer's meaning comes from the state dict and the layer kind only (conv_key / bn_key / src / res / relu of an
``LspgLayerInfo`` row); nothing is read from the library's tap tables or packed weights, so a geometry or packing bug
cannot hide in both the kernel and this reference.

Every layer is written as a sum over *groups*: one source-grid offset (dy, dx) times one 64-channel chunk of the
concatenated sources.  For a stride-1/2 conv the offsets are the 3x3 taps; for nearest-x2 upsample + conv and for the
tail, each output phase (py, px) reads source rows y + floor((py + r - 1) / 2), so the taps of one phase that land on the
same source pixel are summed (in float64 here); the head reads the space-to-depth tensor 0 (channel (py*2+px)*16 + c).
Walking the groups in the kernel's K order, 16 channels per MMA, also gives the accumulator's partial sums, which the
bound needs, and the kernel's own limb products summed exactly, which a second, tighter bound compares against.
``tests/test_layer_reference.py`` ties the chained reference to the float64 oracle (literal upsample + conv).

Quantities are float64 torch tensors on any device; activations are NHWC.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch

KIND_HEAD, KIND_S1, KIND_S2, KIND_UP, KIND_TAIL = range(5)
BN_EPS = 1e-5
U = 2.0 ** -24          # fp32 unit roundoff (round to nearest)
# Tensor-core accumulation model (Hopper wgmma, fp32 accumulate).  One m64nNk16 MMA adds 16 products of 16-bit operands
# (exact: 11 x 11 or 8 x 8 significand bits fit in fp32) to the accumulator C, as one multi-operand addition: the addends
# are aligned to the largest exponent, summed, and the sum is normalised back to fp32 by truncation.  Bits lost when the
# addends are aligned cost at most one fp32 ulp of the sum's magnitude, and the truncating normalisation at most one more,
# so one MMA returns C + sum p within DELTA = 2 * 2^-23 = 2^-22 of (|C| + sum |p|).  Counting one such step per k16 MMA
# (not one per product) is what "K/16 additions" means; the bound sums DELTA (|C| + sum |p|) over the MMAs of the launch
# in the kernel's own K order, with C the float64 partial sum of the limb products before each MMA.  The model assumes the
# adder keeps the aligned addends to within one ulp of the sum; an adder that cut each of the 17 addends to the largest
# one's grid could lose up to 17 ulps per MMA, and tests/test_gpu_layers.py would then fail on the H100.
DELTA = 2.0 ** -22


def _s2d_tap(r: int) -> Tuple[int, int]:
    """Head: input row 2*oy + r - 1 of a stride-2 pad-1 conv = space-to-depth row oy + d, sub-row p.  Returns (p, d)."""
    return (1, -1) if r == 0 else ((0, 0) if r == 1 else (1, 0))


@dataclass
class LayerSpec:
    kind: int
    stride: int                      # source pixel = stride * y + dy
    phases: List[Tuple[int, int]]    # output phases (py, px): up / tail write pixel (2y + py, 2x + px)
    offsets: List[List[Tuple[int, int]]]          # per phase, ascending (dy, dx): the kernel's tap order
    w: List[Dict[Tuple[int, int], torch.Tensor]]  # per phase: offset -> [Cin_total, Cout] float64
    wabs: List[Dict[Tuple[int, int], torch.Tensor]]  # same, sum of |w| over the merged taps
    cin: int
    cout: int
    scale: torch.Tensor              # float64 eval BatchNorm: gamma / sqrt(var + eps)   (1 without BN)
    shift: torch.Tensor              # beta - mean * scale                                (0 without BN)
    mean_scale: torch.Tensor         # |mean * scale|: enters the error of the fp32 shift fold
    relu: bool
    w32: List[Dict[Tuple[int, int], torch.Tensor]]   # per phase: the fp32 tap sums the kernels' weights are cut from
    scale32: torch.Tensor            # the fp32 BatchNorm fold the epilogue applies
    shift32: torch.Tensor


def fp32_presum(w: List[torch.Tensor]) -> torch.Tensor:
    """A merged tap as the weight packer forms it: the fp32 sum of the state-dict taps in (r, s) order."""
    acc = torch.zeros_like(w[0], dtype=torch.float32)
    for t in w:
        acc = acc + t.float()
    return acc


def layer_spec(sd: Dict[str, torch.Tensor], info, mode: str, device=None) -> LayerSpec:
    """``mode`` 'parity': float64 state-dict weights; 'fast': the bf16 weights the FAST kernel multiplies."""
    w = sd[info.conv_key.decode() + ".weight"].to(device)              # [Cout, Cin, 3, 3] fp32
    cout, cin_w = w.shape[0], w.shape[1]
    kind = info.kind
    taps: List[Dict[Tuple[int, int], List[Tuple[int, int]]]] = []        # per phase: offset -> [(r, s)]
    if kind in (KIND_S1, KIND_S2):
        phases = [(0, 0)]
        taps.append({(r - 1, s - 1): [(r, s)] for r in range(3) for s in range(3)})
    elif kind == KIND_HEAD:
        phases = [(0, 0)]
        taps.append({})
        for r in range(3):
            for s in range(3):
                taps[0].setdefault((_s2d_tap(r)[1], _s2d_tap(s)[1]), []).append((r, s))
    else:
        phases = [(py, px) for py in range(2) for px in range(2)]
        for py, px in phases:
            d: Dict[Tuple[int, int], List[Tuple[int, int]]] = {}
            for r in range(3):
                for s in range(3):
                    d.setdefault(((py + r - 1) // 2, (px + s - 1) // 2), []).append((r, s))
            taps.append(d)
    cin = 64 if kind == KIND_HEAD else cin_w
    wd, wa, w32, offs = [], [], [], []
    for z, d in enumerate(taps):
        wz, az, fz = {}, {}, {}
        for off, rs in sorted(d.items()):
            m = torch.zeros(cin, cout, dtype=torch.float64, device=w.device)
            a = torch.zeros_like(m)
            f = torch.zeros(cin, cout, dtype=torch.float32, device=w.device)
            for r, s in rs:
                if kind == KIND_HEAD:
                    p = _s2d_tap(r)[0] * 2 + _s2d_tap(s)[0]
                    rows = slice(p * 16, p * 16 + cin_w)
                else:
                    rows = slice(0, cin)
                m[rows] += w[:, :, r, s].double().t()
                a[rows] += w[:, :, r, s].double().abs().t()
            if kind in (KIND_UP, KIND_TAIL):
                f = fp32_presum([w[:, :, r, s].t() for r, s in rs])
            else:
                f = m.float()                                   # one state-dict tap per entry: exact
            if mode == "fast":
                m = f.bfloat16().double()
                a = m.abs()
            wz[off], az[off], fz[off] = m, a, f
        wd.append(wz)
        wa.append(az)
        w32.append(fz)
        offs.append(sorted(d))
    if info.bn_key:
        k = info.bn_key.decode()
        g, b = sd[k + ".weight"].double().to(w.device), sd[k + ".bias"].double().to(w.device)
        mu, var = sd[k + ".running_mean"].double().to(w.device), sd[k + ".running_var"].double().to(w.device)
        scale = g / torch.sqrt(var + BN_EPS)
        shift = b - mu * scale
        ms = (mu * scale).abs()
        sc32 = g.float() * (1.0 / torch.sqrt(var.float() + BN_EPS))
        sh32 = b.float() - mu.float() * sc32
    else:
        scale = torch.ones(cout, dtype=torch.float64, device=w.device)
        shift = torch.zeros_like(scale)
        ms = torch.zeros_like(scale)
        sc32, sh32 = scale.float(), shift.float()
    return LayerSpec(kind, 2 if kind == KIND_S2 else 1, phases, offs, wd, wa, cin, cout, scale, shift, ms, bool(info.relu),
                     w32, sc32, sh32)


def gather(x: torch.Tensor, n: torch.Tensor, y: torch.Tensor, xx: torch.Tensor, stride: int, dy: int, dx: int,
           ch: slice = slice(None)) -> torch.Tensor:
    """x[n, stride*y + dy, stride*x + dx, ch] with zeros outside the image (the conv's padding)."""
    b, h, w, c = x.shape
    sy, sx = stride * y + dy, stride * xx + dx
    ok = (sy >= 0) & (sy < h) & (sx >= 0) & (sx < w)
    out = x[n, sy.clamp(0, h - 1), sx.clamp(0, w - 1), ch]
    return out * ok.unsqueeze(1).to(out.dtype)


def chunk_order(spec: LayerSpec, z: int, patch_kernel: bool) -> List[Tuple[Tuple[int, int], slice]]:
    """Groups of phase z in the kernel's K order: conv_patch_kernel loads one halo patch per 64-channel chunk and runs all
    taps on it (chunk-major); conv_umma_kernel walks K = (tap, source, channel) (tap-major)."""
    chunks = [slice(c, c + 64) for c in range(0, spec.cin, 64)]
    if patch_kernel:
        return [(off, ch) for ch in chunks for off in spec.offsets[z]]
    return [(off, ch) for off in spec.offsets[z] for ch in chunks]


def k_items(spec: LayerSpec, z: int, patch_kernel: bool) -> List[List[Tuple[Tuple[int, int], slice]]]:
    """The K loop as split-K cuts it: a patch-kernel item is one chunk with all its taps, a per-tap-kernel item one group."""
    order = chunk_order(spec, z, patch_kernel)
    per = len(spec.offsets[z]) if patch_kernel else 1
    return [order[i:i + per] for i in range(0, len(order), per)]


PARITY_WEIGHT_SCALE = 256.0        # include/lspg.h: LSPG_PARITY_WEIGHT_SCALE
LIMB_PRODUCTS = {"parity": [(0, 0), (0, 1), (1, 0)], "fast": [(0, 0)]}   # (activation limb, weight limb) per MMA


def kernel_weights(spec: LayerSpec, z: int, off: Tuple[int, int], ch: slice, mode: str) -> List[torch.Tensor]:
    """The weight operands the kernel multiplies, built from the fp32 tap sums: PARITY the fp16 limbs of w * 2^8,
    FAST bf16(w)."""
    w32 = spec.w32[z][off][ch]
    if mode == "parity":
        ws = w32 * PARITY_WEIGHT_SCALE
        hi = ws.half()
        return [hi.double(), (ws - hi.float()).half().double()]
    return [w32.bfloat16().double()]


def kernel_scale(spec: LayerSpec, mode: str) -> torch.Tensor:
    return spec.scale32.double() / (PARITY_WEIGHT_SCALE if mode == "parity" else 1.0)


@dataclass
class LayerResult:
    value: torch.Tensor      # [P, Cout] float64 layer output (after BN / residual / ReLU; tail: tanh)
    bound: torch.Tensor      # [P, Cout] error bound of the kernel's stored output


def evaluate(spec: LayerSpec, xs: List[torch.Tensor], n, y, xx, z: int, mode: str, geo,
             res: Optional[List[torch.Tensor]] = None) -> Tuple[LayerResult, LayerResult]:
    """The layer at source-grid pixels (n, y, xx) of phase z, two ways.

    ``xs``: the limbs of the concatenated sources the kernel consumed (PARITY [hi, lo], FAST [bf16 value]), NHWC float64;
    ``res``: the limbs of the residual at the output pixels, [P, Cout] each; ``geo``: the launch's ``LspgLayerGeo``.

    Returns (semantic, kernel).  *semantic*: the layer from the float64 state-dict weights (FAST: the bf16 weights) and the
    float64 BatchNorm, with the full bound.  *kernel*: the kernel's own limb products and fp32 BatchNorm fold summed
    exactly, whose bound holds only the fp32 accumulation and the epilogue's roundings: a missing or wrong limb product
    shows up here at any K.
    """
    p = n.shape[0]
    f64 = dict(dtype=torch.float64, device=xs[0].device)
    acc = torch.zeros(p, spec.cout, **f64)        # semantic
    aabs = torch.zeros_like(acc)                  # sum |a| |w| (PARITY: with the operand slack, see bound())
    kacc = torch.zeros_like(acc)                  # the kernel's limb products, exact
    kabs = torch.zeros_like(acc)
    run = torch.zeros_like(acc)                   # sum over MMAs of |C| + sum |p|
    fin = torch.zeros_like(acc)                   # split-K finisher: sum of |prefix sums of the split partials|
    items = k_items(spec, z, geo.kernel == 1)
    for s in range(geo.n_split):
        loc = torch.zeros_like(acc)               # this split's accumulator (starts at zero)
        for item in items[s * geo.split_len:(s + 1) * geo.split_len]:
            for off, ch in item:
                a = [gather(t, n, y, xx, spec.stride, off[0], off[1], ch) for t in xs]
                av = a[0] if len(a) == 1 else a[0] + a[1]
                acc += av @ spec.w[z][off][ch]
                if mode == "parity":
                    aabs += (av.abs() + 2.0 ** -13) @ (spec.wabs[z][off][ch] + 2.0 ** -11)
                else:
                    aabs += av.abs() @ spec.wabs[z][off][ch]
                wk = kernel_weights(spec, z, off, ch, mode)
                for k in range(0, a[0].shape[1], 16):
                    for ia, iw in LIMB_PRODUCTS[mode]:
                        ak, wkk = a[ia][:, k:k + 16], wk[iw][k:k + 16]
                        pa = ak.abs() @ wkk.abs()
                        run += loc.abs() + pa
                        loc += ak @ wkk
                        kabs += pa
        kacc += loc
        if geo.n_split > 1:
            fin += kacc.abs()
    rv = (res[0] if len(res) == 1 else res[0] + res[1]) if res is not None else None
    sem = finish(spec, acc, spec.scale, spec.shift, rv)
    ker = finish(spec, kacc, kernel_scale(spec, mode), spec.shift32.double(), rv)
    return (LayerResult(sem.value, bound(spec, mode, spec.scale, aabs, run, fin, rv, sem.value, operands=True)),
            LayerResult(ker.value, bound(spec, mode, kernel_scale(spec, mode), kabs, run, fin, rv, ker.value, operands=False)))


@dataclass
class _Value:
    value: torch.Tensor


def finish(spec: LayerSpec, acc, scale, shift, res: Optional[torch.Tensor]) -> _Value:
    z = acc * scale + shift
    if spec.kind == KIND_TAIL:
        return _Value(torch.tanh(z))
    v = z + (res if res is not None else 0.0)
    return _Value(torch.relu(v) if spec.relu else v)


def reference_value(spec: LayerSpec, x: torch.Tensor, n, y, xx, z: int, res: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The semantic value alone (float64 state-dict weights), at source-grid pixels (n, y, xx) of phase z."""
    acc = torch.zeros(n.shape[0], spec.cout, dtype=torch.float64, device=x.device)
    for off in spec.offsets[z]:
        acc += gather(x, n, y, xx, spec.stride, off[0], off[1]) @ spec.w[z][off]
    return finish(spec, acc, spec.scale, spec.shift, res).value


def bound(spec: LayerSpec, mode: str, scale, aabs, run, fin, res, v, operands: bool) -> torch.Tensor:
    """Bound on |kernel's stored output - float64 reference| per element, derived from the kernel's arithmetic.

    scale: the scale the reference applies; aabs = A = sum |a| |w|; run = R = sum over the launch's MMAs of |C| + sum |p|
    (C: the accumulator before the MMA, in the kernel's K order, restarting at zero for each split-K range); fin = sum of
    |prefix sums| of the split partials; res: the residual; v: the reference output.
    S = |scale| A + |shift| + |res| bounds every fp32 intermediate of the epilogue.

    Always (``operands=False``: the reference is the kernel's own limb products with its fp32 scale and shift):
      * accumulation: DELTA R (model at DELTA), plus u fin for the finisher's fp32 sum of the split partials.
      * epilogue: fmaf(acc, scale, shift) rounds once, each residual limb add once: <= (1 + limbs) u S.
      * PARITY store: hi = fp16(y), lo = fp16(y - hi) (y - hi is exact): <= 2^-22 |y| + 2^-25.
      * FAST store: bf16 keeps 8 significand bits, so one ulp is at most 2^-7 |y|; the round-to-nearest store is within
        half of that, and the bound allows the full ulp so that a value at a rounding boundary may go either way.
      * tail: no 16-bit store; tanh is 1-Lipschitz and tanhf is within 2 ulp: + 2^-22 |tanh|.
    With ``operands=True`` (the reference is the float64 state-dict layer) also:
      * BatchNorm fold in fp32: scale = gamma * (1 / sqrt(var + eps)) carries <= 4 roundings (4u |scale| A after the
        multiply); shift = beta - mean * scale carries u |shift| + 5u |mean scale|.
      * PARITY operands (activations hi + lo fp16 are read exactly; weights are hi + lo fp16 of w * 2^8):
        the weight limbs carry 22 bits, |w_hi + w_lo - w| <= 2^-22 |w| + 2^-33 (a subnormal lo limb is exact to
        2^-25 / 2^8); the upsample / tail taps are summed in fp32 first, <= 3u sum |w_i| (at most 4 taps merge); the
        missing lo*lo product, |a_lo| <= 2^-11 |a| + 2^-25 and |w_lo| <= 2^-11 |w| + 2^-33.  All are covered by
        (2^-21 + 3u) A with A built from (|a| + 2^-13)(|w| + 2^-11).  FAST multiplies the exact bf16 weights: no term.
    """
    sc = scale.abs()
    shift = spec.shift if operands else spec.shift32.double()
    limbs = 2 if mode == "parity" else 1
    rabs = res.abs() if res is not None else 0.0
    s = sc * aabs + shift.abs() + rabs
    pre = sc * (DELTA * run + U * fin) + (1 + limbs) * U * s
    if operands:
        pre = pre + sc * 4 * U * aabs + U * shift.abs() + 5 * U * spec.mean_scale
        if mode == "parity":
            pre = pre + sc * (2.0 ** -21 + 3 * U) * aabs
    if spec.kind == KIND_TAIL:
        return pre + 2.0 ** -22 * v.abs()
    if mode == "parity":
        return pre + 2.0 ** -22 * (v.abs() + pre) + 2.0 ** -25
    return pre + 2.0 ** -7 * (v.abs() + pre)


def unpack_s2d(s: torch.Tensor, in_nc: int = 13) -> torch.Tensor:
    """Tensor 0 (space-to-depth NHWC [B, H/2, W/2, 64], channel (py*2+px)*16 + c) -> NCHW [B, in_nc, H, W]."""
    b, h2, w2, _ = s.shape
    x = torch.zeros(b, in_nc, 2 * h2, 2 * w2, dtype=s.dtype, device=s.device)
    for py in range(2):
        for px in range(2):
            q = (py * 2 + px) * 16
            x[:, :, py::2, px::2] = s[..., q:q + in_nc].permute(0, 3, 1, 2)
    return x


def pack_s2d(x: torch.Tensor) -> torch.Tensor:
    """NCHW [B, C<=16, H, W] -> space-to-depth NHWC [B, H/2, W/2, 64] (the input packer's layout)."""
    b, c, h, w = x.shape
    s = torch.zeros(b, h // 2, w // 2, 64, dtype=x.dtype, device=x.device)
    for py in range(2):
        for px in range(2):
            q = (py * 2 + px) * 16
            s[..., q:q + c] = x[:, :, py::2, px::2].permute(0, 2, 3, 1)
    return s


def planner_variants(lib, handle, batch: int, height: int, width: int) -> Dict[tuple, List[int]]:
    """(kernel, BN, tail, cluster, split-K) -> layers the planner gives it for this problem size."""
    import ctypes as C
    from livespeechportraits_b200 import _lib
    n = C.c_int()
    _lib.check(lib.lspg_num_layers(handle, C.byref(n)))
    out: Dict[tuple, List[int]] = {}
    for i in range(n.value):
        info, g = _lib.LspgLayerInfo(), _lib.LspgLayerGeo()
        _lib.check(lib.lspg_layer_info_get(handle, i, C.byref(info)))
        _lib.check(lib.lspg_debug_layer_geo(handle, i, batch, height, width, C.byref(g)))
        key = ("patch" if g.kernel == 1 else "umma", g.bn, info.kind == KIND_TAIL, g.cluster, g.n_split > 1)
        out.setdefault(key, []).append(i)
    return out


def grid_pixels(b: int, h: int, w: int, device=None):
    n, y, x = torch.meshgrid(torch.arange(b, device=device), torch.arange(h, device=device), torch.arange(w, device=device),
                             indexing="ij")
    return n.reshape(-1), y.reshape(-1), x.reshape(-1)


def output_pixels(spec: LayerSpec, z: int, y, xx):
    """Output pixel of source-grid pixel (y, x) in phase z."""
    if spec.kind in (KIND_UP, KIND_TAIL):
        py, px = spec.phases[z]
        return 2 * y + py, 2 * xx + px
    return y, xx


def layer_full(spec: LayerSpec, xs: List[torch.Tensor], mode: str, geo, res: Optional[List[torch.Tensor]] = None,
               value_only: bool = False, rows: Optional[int] = None):
    """The whole layer as NHWC [B, Ho, Wo, Cout] (tail: [B, H, W, 3] after tanh), in pixel slices.

    ``xs`` / ``res``: limbs as in ``evaluate`` (full tensors).  Returns the semantic value alone if ``value_only``, else
    (semantic value, its bound, kernel value, its bound)."""
    b, h, w, _ = xs[0].shape
    hs, ws = (h // 2, w // 2) if spec.kind == KIND_S2 else (h, w)
    up = spec.kind in (KIND_UP, KIND_TAIL)
    ho, wo = (2 * hs, 2 * ws) if up else (hs, ws)
    rows = rows or max(4096, (1 << 23) // spec.cout)
    outs = [torch.zeros(b, ho, wo, spec.cout, dtype=torch.float64, device=xs[0].device) for _ in range(1 if value_only else 4)]
    n, y, xx = grid_pixels(b, hs, ws, xs[0].device)
    x = xs[0] if len(xs) == 1 else xs[0] + xs[1]
    for z in range(len(spec.phases)):
        for i in range(0, n.shape[0], rows):
            nn, yy, xq = n[i:i + rows], y[i:i + rows], xx[i:i + rows]
            oy, ox = output_pixels(spec, z, yy, xq)
            r = [t[nn, oy, ox] for t in res] if res is not None else None
            if value_only:
                outs[0][nn, oy, ox] = reference_value(spec, x, nn, yy, xq, z, sum(r) if r is not None else None)
                continue
            sem, ker = evaluate(spec, xs, nn, yy, xq, z, mode, geo, r)
            for t, v in zip(outs, (sem.value, sem.bound, ker.value, ker.bound)):
                t[nn, oy, ox] = v
    return outs[0] if value_only else tuple(outs)
