"""Compile the CUDA extension in-tree for sm_90a (nvcc cross-compiles without a GPU).

``python -m livespeechportraits_b200.build`` or ``build_library()`` produces
``livespeechportraits_b200/liblspg.so`` - a plain C-ABI shared library (include/lspg.h, include/lsph.h, include/lspm.h, include/lspa.h, include/lspl.h, include/lspr.h, include/lspj.h, include/lspv.h), statically linked
against cudart and without a link-time dependency on libcuda (the one driver entry point it needs,
cuTensorMapEncodeTiled, is resolved at run time), so it also loads on a machine without a driver.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.path.join(PKG_DIR, "liblspg.so")
SOURCES = ["lspg.cu", "lsph.cu", "lspm.cu", "lspa.cu", "lspl.cu", "lspr.cu", "lspj.cu", "lspv.cu"]
HEADERS = ["capi.cuh", "bitstream.cuh", "conv_wgmma.cuh", "ptx.cuh", "aux_kernels.cuh", "raster.cuh", "gemm_nt.cuh", os.path.join("..", "..", "include", "lspg.h"),
           os.path.join("..", "..", "include", "lsph.h"), os.path.join("..", "..", "include", "lspm.h"),
           os.path.join("..", "..", "include", "lspa.h"), os.path.join("..", "..", "include", "lspl.h"),
           os.path.join("..", "..", "include", "lspr.h"), os.path.join("..", "..", "include", "lspj.h"),
           os.path.join("..", "..", "include", "lspv.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-shared", "-Xcompiler", "-fPIC",
    "-cudart", "static",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; the CUDA extension cannot be built (there is no CPU fallback)")


def needs_build() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build_library(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB_PATH
    cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB_PATH] + SOURCES
    proc = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + proc.stdout + proc.stderr)
    if verbose:
        sys.stderr.write(proc.stdout + proc.stderr)
    return LIB_PATH


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
