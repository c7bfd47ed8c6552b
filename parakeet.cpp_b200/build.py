"""Builds parakeet.cpp_b200/libparakeet_b200.so IN-TREE with nvcc for sm_90a.

    python parakeet.cpp_b200/build.py [--force]

One translation unit per kernel group (csrc/*.cu), compiled in parallel with
`-gencode arch=compute_90a,code=sm_90a -lineinfo`, linked into one shared
library that exports the C-ABI of include/parakeet_b200.h.  nvcc cross-compiles
without a GPU; the .so is git-ignored.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libparakeet_b200.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall", "-diag-suppress", "550"]
CU = ["mel.cu", "subsample.cu", "gemm_simt.cu", "gemm_tc.cu", "gemm_skinny.cu", "attention.cu", "attention_tc.cu", "attention_mha.cu", "speaker_head.cu", "norm_conv.cu", "ctc.cu", "ctc_beam.cu", "ctc_align.cu",
      "tdt.cu", "stream.cu", "stream_engine.cu", "resample.cu", "engine.cu",
      "kernel_hooks.cu"]
CPP = ["safetensors.cpp", "text.cpp", "nccl_dl.cpp", "lm.cpp"]


def _newer(src_list, out):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(s) > t for s in src_list)


def _headers():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    hs.append(os.path.join(HERE, "..", "include", "parakeet_b200.h"))
    return hs


def _compile(src, force):
    out = os.path.join(OBJ, os.path.basename(src) + ".o")
    if not force and not _newer([src] + _headers(), out):
        return out, ""
    cmd = [NVCC] + NVCC_FLAGS + ["-c", src, "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    return out, r.stderr


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    srcs = [os.path.join(CSRC, f) for f in CU + CPP if os.path.exists(os.path.join(CSRC, f))]
    with ThreadPoolExecutor(max_workers=8) as ex:
        results = list(ex.map(lambda s: _compile(s, force), srcs))
    objs = [o for o, _ in results]
    if verbose:
        for _, log in results:
            if log.strip():
                print(log, file=sys.stderr)
    if force or _newer(objs, LIB):
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-lcudart", "-ldl"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
