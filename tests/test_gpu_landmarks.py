"""Row N7 (SURVEY.md 8f) on the GPU: the landmark post-processing of include/lspl.h against the float64 truth within the
per-element bound derived from the kernel's arithmetic (``landmark_oracle.error_bound``), on the golden cases generated
from demo.py's stage 5, other lengths and a 10-minute clip; determinism; the rasterised maps against the reference's
output; the device chain head-pose loop -> post-processing -> rasteriser -> generator; ``render_to_video`` and
``postprocess_clip``."""
import functools
import json
import os
import types

import numpy as np
import pytest
import torch

from oracle import landmark_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
GOLD_DIR = os.path.join(os.path.dirname(__file__), "golden", "landmarks")
GOLDENS = ["may_672", "obama1_672", "xy_200", "lowermore_200", "mouth_sigma0_150", "head_longer_300_340",
           "feat_longer_340_300", "no_crossing_200", "n1", "n2", "n7", "n41", "pad_200"]
KEYS = ("landmarks", "shoulders", "final_pts3d", "pred_headpose")


def _golden(name):
    g = np.load(os.path.join(GOLD_DIR, name + ".npz"))
    ident = {k: g["id_" + k] for k in O.IDENTITY_KEYS}
    ident["scale"] = np.float64(ident["scale"])
    pad = tuple(int(v) for v in g["image_pad"]) or None
    ref = {"landmarks": g["pred_landmarks"], "shoulders": g["pred_shoulders"], "final_pts3d": g["final_pts3d"],
           "pred_headpose": g["pred_headpose"]}
    return g["pred_Feat"], g["pred_Head"], ident, json.loads(str(g["params"])), pad, ref


def _params(prm):
    from livespeechportraits_b200.landmarks import StageParams
    return StageParams(prm["Feat_smooth_sigma"], prm["AMP_method"], prm["Feat_AMPs"], prm["rot_AMP"], prm["trans_AMP"],
                       prm["Head_smooth_sigma"], prm["shoulder_AMP"])


@functools.lru_cache(maxsize=4)
def _post(id_seed=0, m=37):
    from livespeechportraits_b200.landmarks import Identity, LandmarkPostprocessor
    return LandmarkPostprocessor(Identity(**O.make_identity(id_seed, m)), device=DEV)


def _run(ident, feat, head, prm, pad=None):
    from livespeechportraits_b200.landmarks import Identity, LandmarkPostprocessor
    post = LandmarkPostprocessor(Identity(**ident), device=DEV)
    out = post.run(torch.from_numpy(feat).to(DEV), torch.from_numpy(head).to(DEV), _params(prm), image_pad=pad,
                   return_intermediates=True)
    return dict(zip(KEYS, (t.cpu().numpy() for t in out)))


def _check(got, feat, head, ident, prm, pad, label):
    t = O.truth(feat, head, ident, prm, pad)
    b = O.error_bound(t)
    worst = {}
    for k in KEYS:
        assert got[k].dtype == np.float32 and got[k].shape == t[k].shape, k
        worst[k] = float((np.abs(got[k] - t[k]) / b[k]).max()) if got[k].size else 0.0
    print(f"{label}: nframe {got['landmarks'].shape[0]}, worst error/bound " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    assert max(worst.values()) <= 1.0, worst
    return t, b


@pytest.mark.parametrize("name", GOLDENS)
def test_goldens_within_the_bound(name):
    feat, head, ident, prm, pad, ref = _golden(name)
    got = _run(ident, feat, head, prm, pad)
    _check(got, feat, head, ident, prm, pad, name)
    d = max(float(np.abs(got[k] - ref[k]).max()) for k in ("landmarks", "shoulders"))
    print(f"{name}: max pixel distance to the reference output {d:.3g}")
    assert d < 1e-3


@pytest.mark.parametrize("n_feat,n_head", [(3, 3), (33, 33), (65, 64), (64, 65), (100, 1), (1, 100), (500, 97)])
def test_other_lengths(n_feat, n_head):
    ident = O.make_identity(0, 37)
    feat, head = O.make_tracks(n_feat, n_head, n_feat + n_head)
    got = _run(ident, feat, head, O.MAY)
    _check(got, feat, head, ident, O.MAY, None, f"n_feat {n_feat}, n_head {n_head}")


def test_ten_minute_clip_and_determinism():
    """36,000 frames: a wrong frame index or reduction shows up against the truth somewhere along the clip."""
    ident = O.make_identity(0, 37)
    feat, head = O.make_tracks(36000, 36010, 41)
    post = _post()
    f, h = torch.from_numpy(feat).to(DEV), torch.from_numpy(head).to(DEV)
    first = post.run(f, h, _params(O.MAY), return_intermediates=True)
    got = dict(zip(KEYS, (t.cpu().numpy() for t in first)))
    _check(got, feat, head, ident, O.MAY, None, "10 min")
    for _ in range(2):
        again = post.run(f, h, _params(O.MAY), return_intermediates=True)
        assert all(torch.equal(a, b) for a, b in zip(first, again))


def test_empty_clip_launches_nothing():
    post = _post()
    for nf, nh in ((0, 10), (10, 0), (0, 0)):
        lm, sh = post.run(torch.zeros((nf, 75), device=DEV), torch.zeros((nh, 12), device=DEV), _params(O.MAY))
        assert lm.shape == (0, 73, 2) and sh.shape == (0, 18, 2)


def test_rasterised_maps_match_the_reference_output():
    """The rasteriser truncates to int, so frames where a golden coordinate lies within (bound + |golden - truth|) of an
    integer may differ by one pixel step; every other frame's map equals the oracle rasteriser's map of the golden."""
    from livespeechportraits_b200.generator import Feature2Face_G
    from oracle import raster_oracle as R
    from oracle import f2f_oracle as F
    net = Feature2Face_G(types.SimpleNamespace(isTrain=False, size="normal", n_downsample_G=8, ngf=64, fp16=0),
                         precision="parity")
    net.load_state_dict(F.make_state_dict("normal", "B"))
    net = net.to(DEV).eval()
    checked = skipped = 0
    for name in ("may_672", "pad_200"):
        feat, head, ident, prm, pad, ref = _golden(name)
        got = _run(ident, feat, head, prm, pad)
        t = O.truth(feat, head, ident, prm, pad)
        b = O.error_bound(t)
        fm = net.draw_feature_maps(torch.from_numpy(got["landmarks"]).to(DEV), torch.from_numpy(got["shoulders"]).to(DEV),
                                   (512, 512)).cpu().numpy()
        for k in range(got["landmarks"].shape[0]):
            near = False
            for key in ("landmarks", "shoulders"):
                margin = b[key][k] + np.abs(ref[key][k] - t[key][k])
                near |= bool((np.abs(ref[key][k] - np.round(ref[key][k])) <= margin).any())
            if near:
                skipped += 1
                continue
            assert np.array_equal(fm[k], R.feature_map_tensor(ref["landmarks"][k], (512, 512), ref["shoulders"][k])), (name, k)
            checked += 1
    print(f"raster: {checked} frames bit-equal to the reference output's maps, {skipped} frames with a coordinate near "
          f"an integer")
    assert checked > 0


def test_device_chain_headpose_landmarks_raster_render():
    """HeadposeGenerator -> LandmarkPostprocessor -> draw_feature_maps -> render on one stream with no synchronising
    call; the landmarks agree with the truth computed from the same head-pose track."""
    from livespeechportraits_b200.generator import Feature2Face_G
    from livespeechportraits_b200.headpose import HeadposeGenerator
    from oracle import a2h_oracle as A
    from oracle import f2f_oracle as F
    n = 24
    hopt = A.default_opt()
    gen = HeadposeGenerator(hopt, A.make_state_dict(hopt, "B", 1), device=DEV)
    audio = torch.from_numpy(np.asarray(A.make_audio_feats(hopt.frame_future + n, hopt, 2), np.float32)).to(DEV)
    noise = torch.as_tensor(A.reference_noise(n, 12, 1, seed=0), dtype=torch.float32).to(DEV)
    pre = torch.zeros(12, device=DEV)
    ident = O.make_identity(0, 37)
    feat, _ = O.make_tracks(n, n, 3)
    feat_d = torch.from_numpy(feat).to(DEV)
    net = Feature2Face_G(types.SimpleNamespace(isTrain=False, size="normal", n_downsample_G=8, ngf=64, fp16=0),
                         precision="parity")
    net.load_state_dict(F.make_state_dict("normal", "B"))
    net = net.to(DEV).eval()
    _, cand = F.make_inputs(1, 512, 512, seed=6)
    cand = cand[:1].to(DEV)
    post, prm = _post(), _params(O.MAY)

    def chain():
        head = gen.generate(audio, pre, noise, 0.3)
        lm, sh = post.run(feat_d, head, prm)
        return head, lm, net.render(net.draw_feature_maps(lm, sh, (512, 512)), cand)
    chain()                                       # the generator's first render uploads its weights (a set-up copy)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        head, lm, img = chain()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert img.shape == (n, 3, 512, 512) and torch.isfinite(img).all()
    head_np = head.cpu().numpy().astype(np.float64)
    t = O.truth(feat, head_np, ident, O.MAY)
    b = O.error_bound(t)
    ratio = float((np.abs(lm.cpu().numpy() - t["landmarks"]) / b["landmarks"]).max())
    print(f"chain: {n} frames, worst landmark error/bound {ratio:.3g}")
    assert ratio <= 1.0


def test_render_to_video_takes_device_tracks(tmp_path):
    from livespeechportraits_b200 import render_to_video
    from livespeechportraits_b200.generator import Feature2Face_G
    from oracle import f2f_oracle as F
    net = Feature2Face_G(types.SimpleNamespace(isTrain=False, size="normal", n_downsample_G=8, ngf=64, fp16=0),
                         precision="parity")
    net.load_state_dict(F.make_state_dict("normal", "B"))
    net = net.to(DEV).eval()
    _, cand = F.make_inputs(1, 512, 512, seed=6)
    cand = cand[:1].to(DEV)
    feat, head = O.make_tracks(9, 9, 4)
    lm, sh = _post().run(torch.from_numpy(feat).to(DEV), torch.from_numpy(head).to(DEV), _params(O.MAY))
    a, b = str(tmp_path / "dev.avi"), str(tmp_path / "host.avi")
    render_to_video(net, lm, sh, cand, a, batch=4)
    render_to_video(net, lm.cpu().numpy(), sh.cpu().numpy(), cand, b, batch=4)
    import cv2
    fa, fb = cv2.VideoCapture(a), cv2.VideoCapture(b)
    frames = 0
    while True:
        oka, x = fa.read()
        okb, y = fb.read()
        assert oka == okb
        if not oka:
            break
        assert np.array_equal(x, y)
        frames += 1
    assert frames == 9


def test_postprocess_clip_equals_the_device_call():
    from livespeechportraits_b200.landmarks import postprocess_clip
    feat, head, ident, prm, _, ref = _golden("may_672")
    lm, sh = postprocess_clip(feat, head, ident["mean_pts3d"], ident["std_mean_pts3d"], ident["candidate_eye_brow"],
                              ident["mean_translation"], ident["ref_trans"], ident["shoulder3D"], ident["camera_intrinsic"],
                              ident["scale"], prm["Feat_smooth_sigma"], prm["AMP_method"], prm["Feat_AMPs"], prm["rot_AMP"],
                              prm["trans_AMP"], prm["Head_smooth_sigma"], prm["shoulder_AMP"])
    got = _run(ident, feat, head, prm)
    assert lm.dtype == np.float32 and sh.dtype == np.float32
    assert np.array_equal(lm, got["landmarks"]) and np.array_equal(sh, got["shoulders"])
    assert np.abs(lm - ref["landmarks"]).max() < 1e-3
