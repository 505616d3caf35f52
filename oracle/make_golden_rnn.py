"""Generate tests/golden/rnn/*.npz from the UNMODIFIED reference code - run where the reference checkout exists.

``APC_encoder`` (models/networks.py), ``Audio2Feature`` (models/audio2feature.py) and
``Audio2FeatureModel.generate_sequences`` (models/audio2feature_model.py) are lifted out with ``ast`` and executed
unchanged; ``generate_sequences`` is called with a stand-in ``self`` that holds the ``Audio2Feature`` module and
``device = 'cpu'``.  The script asserts that oracle/rnn_oracle.py's restatement is bit-equal to them, then stores per case
the seeds and shapes (weights and inputs are regenerated from them), a sub-sample of rows of the reference output and of
the float64 truth, and the reference's own max-abs error against the truth over all rows.

    PYTHONDONTWRITEBYTECODE=1 python oracle/make_golden_rnn.py
"""
import ast
import os
import sys
import types
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True
from oracle import rnn_oracle as R  # noqa: E402
from oracle.mel_oracle import REFERENCE_ROOT  # noqa: E402

OUT_DIR = os.path.join(ROOT, "tests", "golden", "rnn")


def _lift(path, wanted, ns, inside=None):
    tree = ast.parse(open(path).read())
    body = tree.body
    if inside:
        body = next(nd for nd in body if isinstance(nd, ast.ClassDef) and nd.name == inside).body
    nodes = [nd for nd in body if isinstance(nd, (ast.FunctionDef, ast.ClassDef)) and nd.name in wanted]
    assert sorted(nd.name for nd in nodes) == sorted(wanted), path
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", SyntaxWarning)
        exec(compile(ast.fix_missing_locations(ast.Module(body=nodes, type_ignores=[])), path, "exec"), ns)


def reference_code():
    from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence
    ns = {"torch": torch, "nn": torch.nn, "np": np, "pack_padded_sequence": pack_padded_sequence,
          "pad_packed_sequence": pad_packed_sequence, "WaveNet": None}
    models = os.path.join(REFERENCE_ROOT, "models")
    _lift(os.path.join(models, "networks.py"), ("APC_encoder",), ns)
    _lift(os.path.join(models, "audio2feature.py"), ("Audio2Feature",), ns)
    _lift(os.path.join(models, "audio2feature_model.py"), ("generate_sequences",), ns, inside="Audio2FeatureModel")
    return ns


def rows_of(n, k):
    return np.unique(np.concatenate([np.arange(0, n, max(1, n // k)), np.arange(max(0, n - 3), n)])).astype(np.int64)


def main():
    ns = reference_code()
    os.makedirs(OUT_DIR, exist_ok=True)
    for recipe in ("A", "B"):
        for T in (2, 37, 1374):
            sd = R.make_apc_state_dict(recipe, 0)
            mel = R.make_mel(T, seed=T)
            m = ns["APC_encoder"](80, 512, 3, False)
            m.load_state_dict(sd, strict=True)
            m.eval()
            with torch.no_grad():
                ref = m.forward(torch.from_numpy(mel)[None], torch.Tensor([T]))[0].numpy()
            mine = R.apc_reference(sd, mel)
            assert np.array_equal(ref, mine), "APC restatement disagrees with the reference"
            truth = R.apc_truth(sd, mel).numpy()
            rows = rows_of(T, 12)
            name = f"apc_{recipe}_T{T}.npz"
            np.savez_compressed(os.path.join(OUT_DIR, name), kind="apc", recipe=recipe, weight_seed=0, input_seed=T, T=T,
                                frame_future=0, rows=rows, ref=ref[rows], truth=truth[rows],
                                ref_err=float(np.abs(ref - truth).max()))
            print(name, "ref err", np.abs(ref - truth).max())
        for n in (2, 36, 1374):
            for ff in (0, 18):
                opt = R.default_mouth_opt(frame_future=ff)
                sd = R.make_mouth_state_dict(opt, recipe, 1)
                feats = R.make_feats(n, seed=n + ff)
                net = ns["Audio2Feature"](types.SimpleNamespace(**vars(opt)))
                net.load_state_dict(sd, strict=True)
                net.eval()
                ref = ns["generate_sequences"](types.SimpleNamespace(Audio2Feature=net, device="cpu"), feats.copy(), opt=opt)
                mine = R.generate_sequences(R.mouth_module(opt, sd), feats, opt)
                assert np.array_equal(ref, mine), "Audio2Mouth restatement disagrees with the reference"
                truth = R.mouth_truth(sd, feats, opt).numpy()
                rows = rows_of(n // 2, 24)
                name = f"mouth_{recipe}_n{n}_ff{ff}.npz"
                np.savez_compressed(os.path.join(OUT_DIR, name), kind="mouth", recipe=recipe, weight_seed=1, input_seed=n + ff,
                                    T=n, frame_future=ff, rows=rows, ref=ref[rows], truth=truth[rows],
                                    ref_err=float(np.abs(ref - truth).max()))
                print(name, "ref err", np.abs(ref - truth).max())


if __name__ == "__main__":
    main()
