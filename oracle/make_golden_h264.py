"""Writes tests/golden/h264/: a few streams of the restatement (oracle/h264_oracle.py) and the planes the libavcodec that
opencv-python bundles decoded from them (tests/libavcodec.py), so the GPU tests keep a decoder pin where that library
is absent.  ``python -m oracle.make_golden_h264`` from the repository root."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import libavcodec  # noqa: E402
from h264_cases import clip  # noqa: E402
from oracle import h264_oracle as H  # noqa: E402

CASES = [
    {"name": "translate_48x64_qp26_gop4", "kind": "translate", "height": 48, "width": 64, "qp": 26, "gop": 4,
     "search": 8, "frames": 6, "seed": 11},
    {"name": "masks_32x48_qp0_gop60", "kind": "masks", "height": 32, "width": 48, "qp": 0, "gop": 60, "search": 4,
     "frames": 3, "seed": 12},
    {"name": "saturated_32x32_qp51_gop1", "kind": "saturated", "height": 32, "width": 32, "qp": 51, "gop": 1,
     "search": 2, "frames": 2, "seed": 13},
    {"name": "noise_16x16_qp10_gop2", "kind": "noise", "height": 16, "width": 16, "qp": 10, "gop": 2, "search": 1,
     "frames": 3, "seed": 14},
]


def main():
    out = os.path.join(ROOT, "tests", "golden", "h264")
    os.makedirs(out, exist_ok=True)
    for c in CASES:
        frames = clip(c["kind"], c["frames"], c["height"], c["width"], seed=c["seed"])
        aus, _, recs, _ = H.encode(frames, qp=c["qp"], gop=c["gop"], search=c["search"])
        dec = libavcodec.decode(aus)
        assert all(np.array_equal(d[k], r[k]) for d, r in zip(dec, recs) for k in range(3)), c["name"]
        open(os.path.join(out, c["name"] + ".h264"), "wb").write(b"".join(aus))
        np.savez_compressed(os.path.join(out, c["name"] + ".npz"),
                            **{f"{p}{i}": d[k] for i, d in enumerate(dec) for k, p in enumerate("yuv")})
    json.dump(CASES, open(os.path.join(out, "cases.json"), "w"), indent=1)
    print(f"wrote {len(CASES)} streams to {out} (libavcodec {libavcodec.decoder_version() >> 16})")


if __name__ == "__main__":
    main()
