"""Build ``libbaybe_b200.so`` (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

Usage: ``python -m baybe_b200.build [--force]``.  nvcc cross-compiles without a GPU.
"""

from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
OUT_DIR = PKG / "_C"
LIB_PATH = OUT_DIR / "libbaybe_b200.so"
STAMP = OUT_DIR / "build.stamp"

SOURCES = ["model.cu", "fused.cu", "wide.cu", "aux_kernels.cu", "acq.cu", "mo.cu", "objective.cu", "nei.cu", "parego.cu", "peer.cu", "stream.cu",
           "boxdec.cu", "nipv.cu", "grad.cu", "objgrad.cu", "nipvgrad.cu", "hvigrad.cu", "gradlarge.cu",
           "objgradlarge.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
]  # cudart is linked statically (nvcc default): the library adopts the caller's current context
# fused.cu holds 35 instantiations of the scoring kernel and is the longest compile by far: its kernels go through the
# back end on several threads (2 min -> 45 s on 8 cores), so that it stays about as long as the other sources together
SOURCE_FLAGS = {"fused.cu": ["-split-compile", "8"]}


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found (set NVCC or put /usr/local/cuda/bin on PATH)")


def _digest() -> str:
    h = hashlib.sha256()
    for p in sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + [PKG.parent / "include" / "baybe_b200.h"]):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    h.update(repr(sorted(SOURCE_FLAGS.items())).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = True) -> Path:
    """Compile every CUDA source into one shared library; returns its path."""
    OUT_DIR.mkdir(exist_ok=True)
    digest = _digest()
    if not force and LIB_PATH.exists() and STAMP.exists() and STAMP.read_text() == digest:
        return LIB_PATH
    nvcc = _nvcc()
    objs = []
    procs = []
    for src in SOURCES:
        obj = OUT_DIR / (src[:-3] + ".o")
        cmd = [nvcc, *NVCC_FLAGS, *SOURCE_FLAGS.get(src, []), "-c", str(CSRC / src), "-o", str(obj)]
        if verbose:
            print(" ".join(cmd), flush=True)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(str(obj))
    for src, pr in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out.decode()}")
    tmp = LIB_PATH.with_suffix(".so.tmp")  # link aside, then rename: a concurrent reader never sees half a library
    cmd = [nvcc, "-shared", "-o", str(tmp), *objs]
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.run(cmd, check=True)
    os.replace(tmp, LIB_PATH)
    STAMP.write_text(digest)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
