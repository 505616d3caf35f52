"""The six C ABIs together (include/lsp[ghmalr].h): every declared function is bound with explicit argument types, every
``*_create`` refuses a device below -1, each module keeps its own last-error message, and (on two GPUs) no call leaves
the calling thread on the handle's device."""
import ctypes as C
import gc
import os
import re
import types

import pytest
import torch

from livespeechportraits_b200 import _lib, headpose
from oracle import a2h_oracle as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PREFIXES = ["lspg", "lsph", "lspm", "lspa", "lspl", "lspr"]


@pytest.mark.parametrize("prefix", PREFIXES)
def test_header_declares_exactly_the_bound_symbols(prefix):
    header = open(os.path.join(ROOT, "include", prefix + ".h")).read()
    declared = set(re.findall(rf"^(?:int|const char\*)\s+({prefix}_\w+)\s*\(", header, flags=re.M))
    assert declared == set(_lib.symbols(prefix)), declared ^ set(_lib.symbols(prefix))
    lib = _lib.load()
    for name in declared:
        assert getattr(lib, name).argtypes is not None, name


def _apc_config():
    cfg = _lib.LsprConfig()
    cfg.kind, cfg.input_dim, cfg.hidden, cfg.num_layers = _lib.LSPR_KIND["apc"], 80, 512, 3
    return cfg


def _create(lib, prefix, device):
    """``<prefix>_create`` with valid arguments apart from ``device``; the handle is destroyed again."""
    h = C.c_void_p()
    args = {"lspg": (0, 64, 8, 13, 3), "lsph": (C.byref(headpose.config_from_opt(A.default_opt())),), "lspm": (512,),
            "lspa": (), "lspl": (), "lspr": (C.byref(_apc_config()),)}[prefix]
    rc = getattr(lib, prefix + "_create")(C.byref(h), *args, device)
    if h:
        getattr(lib, prefix + "_destroy")(h)
    return rc


@pytest.mark.parametrize("prefix", PREFIXES)
def test_create_refuses_a_device_below_minus_one(prefix):
    lib = _lib.load()
    assert _create(lib, prefix, -1) == 0
    assert _create(lib, prefix, -2) == -1                                            # LSPG_EINVAL, not a host-only handle
    assert b"device" in getattr(lib, prefix + "_last_error")()


def test_each_module_keeps_its_own_last_error():
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.lspa_create(None, -1) == -1
    assert lib.lspm_create(C.byref(h), 33, -1) == -1
    assert lib.lspa_last_error() == b"null argument" and b"dim must be" in lib.lspm_last_error()
    cfg = _apc_config()
    cfg.kind = 7
    assert lib.lspr_create(C.byref(h), C.byref(cfg), -1) == -1
    hcfg = headpose.config_from_opt(A.default_opt())
    hcfg.skip_ch = 128
    assert lib.lsph_create(C.byref(h), C.byref(hcfg), -1) == -1
    assert b"kind must be" in lib.lspr_last_error() and b"skip channels" in lib.lsph_last_error()
    with pytest.raises(_lib.LspgError, match="kind must be"):
        _lib.check(-1, "lspr")


def test_cuda_device_refuses_the_cpu_and_indexes_cuda(monkeypatch):
    with pytest.raises(RuntimeError, match="no CPU path: the widget needs an H100"):
        _lib.cuda_device("cpu", "the widget")
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 3)
    assert _lib.cuda_device("cuda", "the widget") == torch.device("cuda", 3)
    assert _lib.cuda_device(torch.device("cuda", 1), "the widget") == torch.device("cuda", 1)


def _handle_on(prefix, dev):
    """A handle on ``dev`` through the package's own classes, after one call that needs the device."""
    if prefix == "lspg":
        from livespeechportraits_b200.generator import Feature2Face_G
        from oracle import raster_oracle as R
        net = Feature2Face_G(types.SimpleNamespace(isTrain=False, size="normal", n_downsample_G=8, ngf=64, fp16=0))
        lm, _ = R.make_landmarks(1, (256, 256), seed=3)
        net.draw_feature_maps(torch.from_numpy(lm).to(dev), None, (256, 256))
        return net
    if prefix == "lsph":
        opt = A.default_opt()
        return headpose.HeadposeGenerator(opt, A.make_state_dict(opt, "A"), device=dev)
    if prefix == "lspm":
        from livespeechportraits_b200.manifold import ManifoldProjector
        from oracle import lle_oracle as M
        return ManifoldProjector(M.make_database(100, 512, seed=1), device=dev)
    if prefix == "lspa":
        from livespeechportraits_b200.audio import MelFrontEnd
        return MelFrontEnd(device=dev)
    if prefix == "lspl":
        from livespeechportraits_b200.landmarks import Identity, LandmarkPostprocessor
        from oracle import landmark_oracle as P
        return LandmarkPostprocessor(Identity(**P.make_identity(0)), device=dev)
    from livespeechportraits_b200.recurrent import ApcEncoder
    from oracle import rnn_oracle as Q
    return ApcEncoder(Q.make_apc_state_dict("A", 0), device=dev)


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two CUDA devices")
@pytest.mark.parametrize("prefix", PREFIXES)
def test_calls_on_another_device_leave_the_current_device_alone(prefix):
    torch.cuda.set_device(0)
    handle = _handle_on(prefix, torch.device("cuda", 1))
    torch.cuda.synchronize(1)
    assert torch.cuda.current_device() == 0
    del handle
    gc.collect()
    assert torch.cuda.current_device() == 0
