"""Generate tests/golden/mel/*.npz by running the UNMODIFIED ``compute_mel_one_sequence`` / ``Audio2Mel`` of the reference.
TEST INFRASTRUCTURE.

Run in the build container (needs /root/reference):  ``python oracle/make_golden_mel.py``

``funcs/utils.py`` and ``funcs/audio_funcs.py`` import librosa, so ``compute_mel_one_sequence`` (:61-83) and ``Audio2Mel``
are lifted out of the files with ``ast`` at run time and executed unchanged (oracle/mel_oracle.py ``reference_functions``;
nothing is copied into this repository), with a ``librosa_mel_fn`` stub that returns the case's basis and a
``torch.stft`` shim that restores torch 1.7's real output.  The restatement in oracle/mel_oracle.py is asserted bit-equal
to them while generating.

Stored per case: the audio (fp32; the shipped 00083.wav samples are a data fixture), the basis, ``winlen`` / ``winstep``,
the reference's output as fp32 (it holds fp32 values in a float64 array), and the largest |reference - float64 truth|.
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import mel_oracle as O  # noqa: E402

# (name, audio: "wav" or (n_samples, seed), basis seed (None: Slaney), winlen, winstep)
CASES = [
    ("mel_00083_wav", "wav", None, 1 / 60, 0.5 / 60),               # the shipped clip: 1374 windows
    ("mel_synth_2s", (32077, 1), None, 1 / 60, 0.5 / 60),           # every kind of test audio, 240 windows
    ("mel_synth_tail_randbasis", (8123, 2), 3, 1 / 60, 0.5 / 60),   # 60 windows, the last ones short; a random basis
    ("mel_synth_one_frame", (300, 4), None, 1 / 60, 0.5 / 60),      # nframe 1: two windows
    ("mel_synth_empty", (200, 5), None, 1 / 60, 0.5 / 60),          # shorter than one frame: no windows
    ("mel_synth_L200", (6000, 6), None, 200 / 16000, 0.5 / 60),     # the shortest clip the right reflection misses
    ("mel_synth_L199", (6000, 7), None, 199 / 16000, 0.5 / 60),     # the right reflection reads clip sample 198
    ("mel_synth_L190_step67", (6000, 8), None, 190 / 16000, 0.25 / 60),   # the shortest clip; step 66.67
]


def case_audio(spec) -> np.ndarray:
    return O.read_wav() if spec == "wav" else O.make_audio(spec[0], spec[1])


def main() -> None:
    out_dir = os.path.join(os.path.dirname(HERE), "tests", "golden", "mel")
    os.makedirs(out_dir, exist_ok=True)
    for name, spec, bseed, winlen, winstep in CASES:
        audio = case_audio(spec)
        basis = O.make_basis(80, bseed)
        ref = O.reference_functions(basis)["compute_mel_one_sequence"](audio, winlen=winlen, winstep=winstep)
        mine = O.compute_mel_one_sequence(audio, basis, winlen=winlen, winstep=winstep)
        assert ref.dtype == np.float64 and ref.shape == (O.n_windows(len(audio)), 80), (name, ref.shape)
        assert np.array_equal(ref, mine), name
        assert np.array_equal(ref, ref.astype(np.float32)), name
        frame_len = int(16000 * winlen)
        err = 0.0
        if ref.shape[0]:
            t = O.logmel_truth(audio, basis, frame_len=frame_len, step=16000 * winstep)
            err = float(np.abs(ref - t["out"]).max())
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), audio=audio, basis=basis, winlen=winlen, winstep=winstep,
                            out=ref.astype(np.float32), err_truth=err)
        print(f"{name}: {len(audio)} samples, {ref.shape[0]} windows, max|reference - float64 truth| {err:.3g}")


if __name__ == "__main__":
    main()
