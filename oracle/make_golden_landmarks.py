"""Generate tests/golden/landmarks/*.npz by running demo.py's UNMODIFIED stage-5 statements.  TEST INFRASTRUCTURE.

Run in the build container (needs the reference checkout):  ``python oracle/make_golden_landmarks.py``

``funcs/utils.py`` imports librosa, sklearn and tqdm, so, as oracle/make_golden_mel.py does, the functions stage 5
calls are lifted out of the file with ``ast`` and executed unchanged (oracle/landmark_oracle.py
``reference_functions``); the statements between demo.py's ``#### 5.`` and ``#### 6.`` markers are lifted out of its
``__main__`` block the same way (``reference_stage5``).  Nothing is copied into this repository.  The restatement
``landmark_oracle.stage5`` is asserted bit-equal to them while generating.

Stored per case: the identity, the tracks, the parameters, image_pad, and the reference's ``pred_landmarks``,
``pred_shoulders`` (image_pad added in fp32 when the case has one), ``final_pts3d`` and ``pred_headpose[:nframe]``.
"""
from __future__ import annotations

import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import landmark_oracle as O  # noqa: E402

XY = dict(O.MAY, AMP_method="XY", Feat_AMPs=[1.8, 2.2])
LOWER_MORE = dict(O.MAY, AMP_method="LowerMore", Feat_AMPs=[1.2, 1.6, 1.0, 2.0, 2.4, 1.5])
SIGMA0 = dict(O.OBAMA1, Feat_smooth_sigma=0)

# (name, params, n_feat, n_head, track seed, lip crossing offset, image_pad, identity (seed, m))
CASES = [
    ("may_672", O.MAY, 672, 672, 1, 0.1, None, (0, 37)),
    ("obama1_672", O.OBAMA1, 672, 672, 2, 0.1, None, (1, 37)),
    ("xy_200", XY, 200, 200, 3, 0.1, None, (0, 37)),
    ("lowermore_200", LOWER_MORE, 200, 200, 4, 0.1, None, (0, 37)),
    ("mouth_sigma0_150", SIGMA0, 150, 150, 5, 0.1, None, (0, 5)),
    ("head_longer_300_340", O.MAY, 300, 340, 6, 0.1, None, (0, 37)),
    ("feat_longer_340_300", O.MAY, 340, 300, 7, 0.1, None, (0, 37)),
    ("no_crossing_200", O.MAY, 200, 200, 8, -0.5, None, (0, 37)),
    ("n1", O.MAY, 1, 1, 9, 0.1, None, (0, 37)),
    ("n2", O.MAY, 2, 2, 10, 0.1, None, (0, 37)),
    ("n7", O.MAY, 7, 7, 11, 0.1, None, (0, 3)),
    ("n41", O.MAY, 41, 41, 12, 0.1, None, (0, 37)),
    ("pad_200", O.MAY, 200, 200, 13, 0.1, (12, 3, 7, 20), (2, 37)),
]


def lip_crossings(feat, ident, prm, nframe):
    """Per frame, how many inner-lip pairs cross before the fix, and the smallest |lower - upper| of the clip."""
    pts = np.zeros([nframe, 73, 3])
    pts[:, O.MOUTH_INDICES] = feat.reshape(-1, 25, 3)[:nframe]
    if prm["Feat_smooth_sigma"] != 0:
        pts[:, 46:64] = O.gaussian_filter1d(pts[:, 46:64].copy().reshape(-1, 54), prm["Feat_smooth_sigma"], axis=0).reshape(-1, 18, 3)
    pts = O.mouth_pts_AMP(pts, True, prm["AMP_method"], prm["Feat_AMPs"]) + ident["mean_pts3d"]
    diff = pts[:, O.LOWER_INNER, 1] - pts[:, O.UPPER_INNER, 1]
    return (diff > 0).sum(axis=1), float(np.abs(diff).min())


def main() -> None:
    warnings.simplefilter("ignore", SyntaxWarning)
    out_dir = os.path.join(os.path.dirname(HERE), "tests", "golden", "landmarks")
    os.makedirs(out_dir, exist_ok=True)
    for name, prm, n_feat, n_head, seed, cross, pad, (id_seed, m) in CASES:
        ident = O.make_identity(id_seed, m)
        feat, head = O.make_tracks(n_feat, n_head, seed, cross)
        nframe = min(n_feat, n_head)
        ref = O.reference_stage5(feat, head, ident, prm)
        if pad is not None:
            top, bottom, left, right = pad
            ref["pred_shoulders"][:, :, 0] += right - left
            ref["pred_shoulders"][:, :, 1] += top - bottom
        mine = O.stage5(feat, head, ident, prm, image_pad=pad)
        for k in ref:
            assert ref[k].dtype == np.float32 and np.array_equal(ref[k], mine[k]), (name, k)
        count, margin = lip_crossings(feat, ident, prm, nframe)
        assert margin > 1e-6, (name, margin)          # the crossing decision is far from a tie
        if name in ("may_672", "obama1_672", "xy_200", "lowermore_200", "mouth_sigma0_150"):
            assert (count == 3).any() and ((count == 2) | (count == 1)).any(), name
        if name.startswith("no_crossing"):
            assert not (count == 3).any(), name
        t = O.truth(feat, head, ident, prm, pad)
        err = float(np.abs(ref["pred_landmarks"] - t["landmarks"]).max())
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), pred_Feat=feat, pred_Head=head,
                            params=json.dumps(prm), image_pad=np.array(pad if pad is not None else [], np.int64),
                            pred_landmarks=ref["pred_landmarks"], pred_shoulders=ref["pred_shoulders"],
                            final_pts3d=ref["final_pts3d"], pred_headpose=ref["pred_headpose"][:nframe],
                            **{"id_" + k: np.asarray(ident[k]) for k in O.IDENTITY_KEYS})
        print(f"{name}: nframe {nframe}, fixed frames {(count == 3).sum()}, two-of-three {(count == 2).sum()}, "
              f"max|reference - float64 truth| landmarks {err:.3g} px")


if __name__ == "__main__":
    main()
