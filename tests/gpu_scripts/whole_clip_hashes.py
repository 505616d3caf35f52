"""Fingerprint the whole-clip outputs of demo.py stages 1-4 on the GPU, so two versions of the library can be compared bit
for bit.

    python tests/gpu_scripts/whole_clip_hashes.py [--out hashes.json]

Uses only the public Python API, so the same file runs against any version of the package that it is placed in.  With
seeded synthetic weights (rnn_oracle / a2h_oracle recipe B) and seeded synthetic audio of two lengths - the length of
00083.wav (183,296 samples: 1,374 mel windows, 687 head-pose audio rows, 672 frames) and 10 minutes - it chains
MelFrontEnd.logmel -> ApcEncoder.forward (cluster 8) -> MouthGenerator.generate and HeadposeGenerator.generate, and prints
ONE JSON line with the shape and the sha256 of the bytes of:
  * MelFrontEnd.logmel;
  * ApcEncoder.forward at cluster 8 and 16;
  * MouthGenerator.generate;
  * HeadposeGenerator.generate at cluster 1 and 8 with return_params (the predictions and the network outputs).
Card name and power limit come from a read-only nvidia-smi query.  Writes only ``--out`` when given.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from lle_bench import card  # noqa: E402
from livespeechportraits_b200.audio import MelFrontEnd  # noqa: E402
from livespeechportraits_b200.headpose import HeadposeGenerator  # noqa: E402
from livespeechportraits_b200.recurrent import ApcEncoder, MouthGenerator  # noqa: E402
from oracle import a2h_oracle as A  # noqa: E402
from oracle import mel_oracle as W  # noqa: E402
from oracle import rnn_oracle as R  # noqa: E402

CLIPS = (("00083.wav length", 183_296), ("10 min", 600 * 16_000))


def fingerprint(t: torch.Tensor) -> dict:
    a = t.detach().cpu().contiguous().numpy()
    return {"shape": list(a.shape), "sha256": hashlib.sha256(a.tobytes()).hexdigest()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    name, limit = card()
    mopt, hopt = R.default_mouth_opt(), A.default_opt()
    front = MelFrontEnd(W.make_basis(80), device=dev)
    enc = ApcEncoder(R.make_apc_state_dict("B", 0), device=dev)
    mouth = MouthGenerator(mopt, R.make_mouth_state_dict(mopt, "B", 0), device=dev)
    head = HeadposeGenerator(hopt, A.make_state_dict(hopt, "B", 1), device=dev)
    pre = torch.zeros(12, device=dev)
    res = {"card": name, "power_limit": limit, "clips": {}}
    for label, n_samples in CLIPS:
        r = {}
        mel = front.logmel(torch.from_numpy(W.make_audio(n_samples, seed=1)).to(dev))
        r["logmel"] = fingerprint(mel)
        feats = None
        for cl in (8, 16):
            out = enc.forward(mel, cluster=cl)
            r[f"apc_cluster{cl}"] = fingerprint(out)
            feats = out if cl == 8 else feats
        r["mouth"] = fingerprint(mouth.generate(feats))
        rows = feats.view(-1, 2 * feats.shape[1])
        nframe = rows.shape[0] - hopt.frame_future
        noise = torch.randn((nframe, 12), generator=torch.Generator().manual_seed(0)).to(dev)
        for cl in (1, 8):
            pred, params = head.generate(rows, pre, noise, 0.3, return_params=True, cluster=cl)
            r[f"headpose_cluster{cl}_pred"] = fingerprint(pred)
            r[f"headpose_cluster{cl}_params"] = fingerprint(params)
        res["clips"][label] = r
    line = json.dumps(res)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
