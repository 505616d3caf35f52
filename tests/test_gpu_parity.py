"""Parity of the CUDA path (through the C ABI, via the drop-in module) against the oracle and the golden
fixtures generated from the reference module.  Tolerance: 1e-3 max-abs on the fp32 [B,3,H,W] output in PARITY
mode (BASELINE.json north_star); FAST (pure bf16 operands) is reported and loosely bounded."""
import glob
import os
import types

import numpy as np
import pytest
import torch

from oracle import f2f_oracle as O

pytestmark = pytest.mark.gpu
TOL = 1e-3
GOLDEN = sorted(p for p in glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.npz"))
                if not os.path.basename(p).startswith(("raster_", "a2h_")))      # raster_*: tests/test_raster_oracle.py


def opt(size):
    return types.SimpleNamespace(isTrain=False, size=size, n_downsample_G=8, ngf=64, fp16=0)


_CACHE = {}


def get_net(variant, recipe):
    from livespeechportraits_b200.generator import Feature2Face_G
    key = (variant, recipe)
    if key not in _CACHE:
        _CACHE.clear()                      # one resident network at a time
        net = Feature2Face_G(opt(variant), precision="parity")
        sd = O.make_state_dict(variant, recipe)
        net.load_state_dict(sd, strict=True)
        _CACHE[key] = (net.cuda().eval(), sd)
    return _CACHE[key]


def test_native_library_is_the_path():
    from livespeechportraits_b200 import _lib
    assert os.path.exists(_lib.library_path())
    net, _ = get_net("normal", "A")
    net(torch.zeros(1, 13, 256, 256, device="cuda"))
    assert net.launches_per_forward() >= 47        # input packer + 46 convs (+ split-K finishers at this size)
    with open("/proc/self/maps") as f:
        assert "liblspg.so" in f.read()


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_parity_mode_matches_reference_golden(path):
    g = np.load(path)
    variant, recipe = str(g["variant"]), str(g["recipe"])
    b, h, w, st = int(g["batch"]), int(g["height"]), int(g["width"]), int(g["stride"])
    net, sd = get_net(variant, recipe)
    fm, cand = O.make_inputs(b, h, w)
    out = net(torch.cat([fm, cand], 1).cuda()).cpu()
    err = np.abs(out[:, :, ::st, ::st].numpy() - g["out_sub"]).max()
    print(f"{os.path.basename(path)}: max|cuda - reference| on the golden sub-sample = {err:.3g}")
    assert err <= TOL
    assert out.shape == (b, 3, h, w) and out.dtype == torch.float32 and float(out.abs().max()) < 1.0
    # the two skip-path activations the fixture carries (e1 after the first down block, d1 before the tail)
    rows = net.layer_table(h, w)
    tail = rows[-1]
    for name, tid in (("e1", tail["src"][0]), ("d1", tail["src"][1])):
        t = (net.debug_read_tensor(tid, b, h, w, 0).float() + net.debug_read_tensor(tid, b, h, w, 1).float())
        t = t.permute(0, 3, 1, 2)[:, ::8, ::st * 2, ::st * 2].numpy()
        ref = g[name + "_sub"]
        assert np.abs(t - ref).max() <= 2e-3 * max(1.0, np.abs(ref).max()), name


@pytest.mark.parametrize("variant,recipe,batch,size", [
    ("normal", "A", 3, 256), ("normal", "B", 1, 512), ("large", "A", 2, 256), ("large", "B", 1, 256),
    ("normal", "B", 8, 512),      # BASELINE.json configs[2]: Obama1 (normal), batch 8, 512x512
    ("large", "A", 1, 512),       # BASELINE.json configs[1]: May (large), single frame
])
def test_parity_mode_matches_oracle_full_output(variant, recipe, batch, size):
    net, sd = get_net(variant, recipe)
    fm, cand = O.make_inputs(batch, size, size, seed=11)
    x = torch.cat([fm, cand], 1)
    out = net(x.cuda()).cpu()
    check = [0] if batch <= 2 else [0, batch - 1]           # the oracle costs ~0.5 s per 512x512 frame on the host
    for i in check:
        ref = O.generator_forward(sd, x[i:i + 1], variant)
        err = (out[i:i + 1] - ref).abs().max().item()
        print(f"{variant} {recipe} B{batch} {size}: frame {i} max|cuda - oracle| = {err:.3g}")
        assert err <= TOL


@pytest.mark.parametrize("variant", ["normal", "large"])
def test_fast_mode_error_is_bf16_sized(variant):
    net, sd = get_net(variant, "A")
    fm, cand = O.make_inputs(1, 512, 512)
    x = torch.cat([fm, cand], 1)
    ref = O.generator_forward(sd, x, variant)
    out = net.render(x.cuda(), None, precision="fast").cpu()
    err = (out - ref).abs().max().item()
    print(f"{variant} FAST (bf16 operands): max|cuda - oracle| = {err:.3g} (contract 1e-3 is met by PARITY mode only)")
    assert err <= 3e-2


def test_zero_in_zero_out_known_answer():
    net, _ = get_net("normal", "A")
    z = torch.zeros(2, 13, 256, 256, device="cuda")
    for mode in ("parity", "fast"):
        assert float(net.render(z, None, precision=mode).abs().max()) == 0.0


def test_determinism_batch_independence_and_permutation():
    net, _ = get_net("normal", "B")
    fm, cand = O.make_inputs(4, 256, 256, seed=3)
    fm[1:] = torch.roll(fm[1:], 1, 2)
    x = torch.cat([fm, cand], 1).cuda()
    a = net(x)
    b = net(x)
    assert torch.equal(a, b)                                       # bit-reproducible
    perm = torch.tensor([2, 0, 3, 1], device="cuda")
    assert torch.equal(net(x[perm]), a[perm])                      # frames are independent batch items (same plan: bit-exact)
    # a different batch size may choose different tiles / split-K factors (fp32 summation order), so across batch
    # sizes independence holds to fp32 rounding, far inside the 1e-3 contract
    assert (net(x[1:2]) - a[1:2]).abs().max().item() <= 5e-5       # a frame does not depend on its batch (split-K factors may differ)
    assert (net(x[:3]) - a[:3]).abs().max().item() <= 5e-5         # ragged batch (3 of a 4-image tile group)


def test_fused_concat_and_candidate_broadcast():
    net, _ = get_net("normal", "B")
    fm, cand = O.make_inputs(3, 256, 256)
    x = torch.cat([fm, cand], 1).cuda()
    a = net(x)
    b = net.render(fm.cuda(), cand[:1].cuda())                      # demo.py:266 reuses one candidate tensor
    c = net.render(fm.cuda(), cand.cuda())
    assert torch.equal(a, b) and torch.equal(a, c)
    pre = torch.full((3, 3, 256, 256), 7.0, device="cuda")
    d = net.render(fm.cuda(), cand[:1].cuda(), out=pre)
    assert d.data_ptr() == pre.data_ptr() and torch.equal(pre, a)


def test_size_generality_1024():
    # BASELINE.json configs[4]: same weights on a 1024x1024 grid (fully convolutional)
    net, sd = get_net("normal", "A")
    fm, cand = O.make_inputs(1, 1024, 1024, seed=2)
    x = torch.cat([fm, cand], 1)
    out = net(x.cuda()).cpu()
    ref = O.generator_forward(sd, x, "normal")
    assert (out - ref).abs().max().item() <= TOL
    fm2, cand2 = O.make_inputs(1, 512, 256, seed=2)              # non-square
    x2 = torch.cat([fm2, cand2], 1)
    assert (net(x2.cuda()).cpu() - O.generator_forward(sd, x2, "normal")).abs().max().item() <= TOL


def test_error_behaviour_on_device():
    from livespeechportraits_b200._lib import LspgError
    net, _ = get_net("normal", "A")
    with pytest.raises(LspgError):
        net(torch.zeros(1, 13, 300, 256, device="cuda"))
    with pytest.raises(TypeError):
        net(torch.zeros(1, 13, 256, 256, device="cuda", dtype=torch.float16))
    with pytest.raises(ValueError):
        net(torch.zeros(1, 12, 256, 256, device="cuda"))


def test_weight_reload_and_dataparallel_wrap():
    from livespeechportraits_b200.generator import Feature2Face_G
    net = Feature2Face_G(opt("normal"), precision="parity").cuda()
    wrapped = torch.nn.DataParallel(net, [0]).eval()               # what networks.init_net does with gpu_ids=[0]
    fm, cand = O.make_inputs(1, 256, 256)
    x = torch.cat([fm, cand], 1)
    for recipe in ("A", "B"):
        sd = O.make_state_dict("normal", recipe)
        wrapped.load_state_dict({"module." + k: v for k, v in sd.items()}, strict=False)
        out = wrapped(x.cuda()).cpu()
        assert (out - O.generator_forward(sd, x, "normal")).abs().max().item() <= TOL


def test_fused_tensor2im_uint8_output():
    """lspg_forward_image = generator + util.tensor2im (util/util.py:19-42) in the tail kernel's epilogue."""
    net, sd = get_net("normal", "B")
    fm, cand = O.make_inputs(2, 256, 256, seed=4)
    x = torch.cat([fm, cand], 1)
    f32 = net(x.cuda())
    u8 = net.render_image(x.cuda(), None)
    assert u8.shape == (2, 256, 256, 3) and u8.dtype == torch.uint8
    # identical arithmetic to applying the reference post-processing to the fp32 frames of the same kernels: bit-exact
    assert np.array_equal(u8.cpu().numpy(), O.tensor2im(f32.cpu()))
    # against the oracle's frames: the fp32 values differ by <= 1e-3, i.e. at most one grey level where a value sits on an
    # integer boundary
    ref = O.tensor2im(O.generator_forward(sd, x, "normal"))
    d = np.abs(u8.cpu().numpy().astype(np.int16) - ref.astype(np.int16))
    assert d.max() <= 1 and (d != 0).mean() < 0.02


def test_clip_renderer_pipeline_matches_direct_calls():
    from livespeechportraits_b200.pipeline import ClipRenderer
    net, _ = get_net("normal", "B")
    fm, cand = O.make_inputs(5, 256, 256, seed=6)
    fm_host = fm.pin_memory()
    direct = net.render(fm.cuda(), cand[:1].cuda()).cpu()
    out_host = torch.empty((5, 3, 256, 256), dtype=torch.float32).pin_memory()
    ClipRenderer(net, batch=2).render_clip(fm_host, cand[:1].cuda(), out_host)     # ragged last batch of 1
    # batches of 2 and 5 frames may use different split-K factors on the sub-16x16 layers (different fp32 summation order)
    assert (out_host - direct).abs().max().item() <= 5e-5
    img_host = torch.empty((5, 256, 256, 3), dtype=torch.uint8).pin_memory()
    ClipRenderer(net, batch=2, uint8=True).render_clip(fm_host, cand[:1].cuda(), img_host)
    d = np.abs(img_host.numpy().astype(np.int16) - O.tensor2im(direct).astype(np.int16))
    assert d.max() <= 1


@pytest.mark.parametrize("recipe,batch", [("A", 64), ("B", 64), ("A", 32), ("B", 32), ("A", 16), ("B", 16)])
def test_large_512_at_the_benchmarked_batch_sizes(recipe, batch):
    """The plan bench.py times (large, 512x512, 32 frames per step by default; 64 and 16 = other tile/wave choices of layer_geo) is the plan
    that is gated: first, middle and last frame of the batch against the oracle at the 1e-3 contract, recipe A and the
    amplifying recipe B, plus the fused-tensor2im uint8 output of the same plan."""
    net, sd = get_net("large", recipe)
    fm, cand = O.make_inputs(batch, 512, 512, seed=21)
    for i in range(1, batch):                                  # distinct frames (make_inputs repeats one candidate set)
        fm[i] = torch.roll(fm[i], shifts=(3 * i, 5 * i), dims=(1, 2))
    x_dev_fm, x_dev_cand = fm.cuda(), cand[:1].cuda()
    out = net.render(x_dev_fm, x_dev_cand).cpu()
    u8 = net.render_image(x_dev_fm, x_dev_cand).cpu().numpy()
    worst = 0.0
    for i in (0, batch // 2, batch - 1):
        x = torch.cat([fm[i:i + 1], cand[:1]], 1)
        ref = O.generator_forward(sd, x, "large")
        err = (out[i:i + 1] - ref).abs().max().item()
        worst = max(worst, err)
        assert err <= TOL, (recipe, batch, i, err)
        d = np.abs(u8[i].astype(np.int16) - O.tensor2im(ref)[0].astype(np.int16))
        assert d.max() <= 1
    assert np.array_equal(u8, O.tensor2im(out))               # same kernels, post-processing fused: bit-exact
    print(f"large {recipe} B{batch} 512: worst of frames 0/{batch // 2}/{batch - 1}: max|cuda - oracle| = {worst:.3g} "
          f"(margin {TOL / max(worst, 1e-12):.1f}x)")


def test_graph_is_captured_once_and_io_pointers_are_patched():
    """One CUDA graph per plan: calls with fresh output tensors / other inputs patch two kernel nodes
    (cudaGraphExecKernelNodeSetParams) instead of re-capturing (round-1 finding: the cache was keyed on raw pointers)."""
    net, sd = get_net("normal", "B")
    fm, cand = O.make_inputs(2, 256, 256, seed=8)
    fm_d, cand_d = fm.cuda(), cand[:1].cuda()
    first = net.render(fm_d, cand_d)
    s0 = net.graph_stats()
    held = [net.render(fm_d, cand_d) for _ in range(40)]                 # the caller keeps every output alive
    fm2 = fm_d.clone()
    held.append(net.render(fm2, cand_d))
    u8 = net.render_image(fm2, cand_d)                                   # same plan, uint8 tail output
    s1 = net.graph_stats()
    assert s1["recaptures"] == 0
    assert s1["captures"] == s0["captures"]                              # nothing was captured again
    assert s1["io_updates"] - s0["io_updates"] >= 41
    assert len({t.data_ptr() for t in held}) == len(held)
    assert all(torch.equal(t, first) for t in held)
    assert np.array_equal(u8.cpu().numpy(), O.tensor2im(first.cpu()))
    # odd-offset views go through an aligned temporary
    big = torch.empty(2 * 3 * 256 * 256 + 1, device="cuda")
    odd = big[1:].view(2, 3, 256, 256)
    assert odd.data_ptr() % 8 == 4
    assert torch.equal(net.render(fm_d, cand_d, out=odd), first)
    with pytest.raises(ValueError):
        net.render(fm_d, cand_d, out=torch.empty(2, 3, 256, 256))       # CPU `out`


def test_forward_refuses_incomplete_weights():
    import ctypes as C
    from livespeechportraits_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.lspg_create(C.byref(h), 0, 64, 8, 13, 3, 0) == 0
    w = torch.randn(64, 13, 3, 3)
    arr = (_lib.LspgTensor * 1)()
    arr[0].name = b"netG.model.model.0.weight"
    arr[0].data = C.cast(w.data_ptr(), C.POINTER(C.c_float))
    arr[0].numel = w.numel()
    assert lib.lspg_load_weights(h, arr, 1) == 0                           # strict=False: a partial dict loads
    need = C.c_size_t()
    assert lib.lspg_workspace_bytes(h, 1, 256, 256, 1, C.byref(need)) == 0
    ws = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    x = torch.zeros(1, 13, 256, 256, device="cuda")
    out = torch.empty(1, 3, 256, 256, device="cuda")
    rc = lib.lspg_forward(h, x.data_ptr(), 13 * 256 * 256, x.data_ptr() + 4 * 256 * 256, 13 * 256 * 256, out.data_ptr(), 1, 256, 256,
                          ws.data_ptr(), ws.numel(), 1, None)
    assert rc == -4 and b"never loaded" in lib.lspg_last_error()           # LSPG_ESTATE, not black frames
    lib.lspg_destroy(h)
