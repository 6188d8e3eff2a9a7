"""Builds libfilm_b200.so in-tree with nvcc for sm_90a (no torch, no cmake).

    python -m frame_interpolation_b200.build [--force] [--verbose]

The library links cudart statically and resolves cuTensorMapEncodeTiled through
cudaGetDriverEntryPoint, so it has no link-time dependency on libcuda and loads on a
box without a GPU (calls then fail with status 2 -- there is no CPU fallback).
"""
from __future__ import annotations

import argparse
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SOURCES = ["film_engine.cu", "film_kernels.cu", "film_conv_tc.cu", "film_conv3x3_tc.cu"]
HEADERS = ["film_common.cuh", "film_conv.h", "film_kernels.h", "film_pack.h", "film_tc_ptx.cuh", os.path.join("..", "..", "include", "film_b200.h")]
LIB = os.path.join(HERE, "libfilm_b200.so")
STAMP = os.path.join(HERE, "_build", "stamp")
# ptxas remark (C75xx) for a kernel whose wgmma instructions it had to serialise; the build fails on it
SERIALIZED = "wgmma.mma_async instructions are serialized"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _digest(extra: str) -> str:
    h = hashlib.sha256(extra.encode())
    for f in SOURCES + HEADERS:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    flags = list(NVCC_FLAGS)
    # 16-bit split format of activations and weights: fp16 (default: 11-bit planes, which is what makes the
    # single-pass stages of the precision plan possible) or bf16 (FILM_SPLIT=bf16: 8-bit planes, every stage
    # must then run three-pass -- set the option onepass_mask = 0)
    if os.environ.get("FILM_SPLIT", "fp16") == "fp16":
        flags.append("-DFILM_SPLIT_FP16")
    if verbose:
        flags += ["-Xptxas", "-v"]
    dig = _digest(" ".join(flags))
    if not force and os.path.exists(LIB) and os.path.exists(STAMP):
        with open(STAMP) as f:
            if f.read().strip() == dig:
                return LIB
    os.makedirs(os.path.dirname(STAMP), exist_ok=True)
    nvcc = _nvcc()
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(HERE, "_build", src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [nvcc, *flags, "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    serialized = []
    for cmd, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stderr.write(out)
        if p.returncode:
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
        serialized += [ln for ln in out.splitlines() if SERIALIZED in ln]
    if serialized:
        # ptxas let each wgmma wait for the previous one to finish: a silent loss of most of the tensor-core rate
        raise RuntimeError("ptxas serialised wgmma:\n" + "\n".join(serialized))
    link = [nvcc, "-shared", "-o", LIB, *objs, "-cudart", "static", "-Xlinker", "-z,defs", "-lpthread", "-ldl", "-lrt"]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if verbose or r.returncode:
        sys.stderr.write(r.stdout)
    if r.returncode:
        raise RuntimeError("link failed: " + " ".join(link))
    with open(STAMP, "w") as f:
        f.write(dig)
    return LIB


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    a = ap.parse_args()
    print(build(a.force, a.verbose))
