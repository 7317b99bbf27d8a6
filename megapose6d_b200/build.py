"""Build libmpx.so (the C-ABI CUDA library) in-tree for sm_90a (H100).

`python -m megapose6d_b200.build` or `build_library()`; nvcc cross-compiles without a GPU.
The shared object lands next to the sources (megapose6d_b200/csrc/libmpx.so), where the package loads it
from the source tree.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

CSRC = Path(__file__).resolve().parent / "csrc"
LIB_PATH = CSRC / "libmpx.so"
SOURCES = ["abi.cu", "conv_wgmma.cu", "net.cu", "detector_net.cu", "detector_heads.cu", "raster.cu", "geom.cu", "crop.cu", "bop_eval.cu", "teaser.cu"]
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    *ARCH_FLAGS,
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _digest() -> str:
    h = hashlib.sha256()
    for path in sorted(CSRC.glob("*.cu")) + sorted(CSRC.glob("*.cuh")):
        h.update(path.name.encode())
        h.update(path.read_bytes())
    h.update((CSRC.parent.parent / "include" / "mpx.h").read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build_library(force: bool = False, verbose: bool = False) -> Path:
    stamp = CSRC / ".libmpx.stamp"
    digest = _digest()
    if not force and LIB_PATH.exists() and stamp.exists() and stamp.read_text() == digest:
        return LIB_PATH
    nvcc = _nvcc()
    objs = []

    def compile_one(src: str) -> Path:
        obj = CSRC / (src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(CSRC / src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
            print(" ".join(cmd), flush=True)
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{res.stdout}\n{res.stderr}")
        if verbose:
            print(res.stderr, flush=True)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    link = [nvcc, "-shared", *ARCH_FLAGS, "-o", str(LIB_PATH),
            *map(str, objs), "-Xcompiler", "-fPIC", "-cudart", "static"]
    res = subprocess.run(link, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    stamp.write_text(digest)
    return LIB_PATH


if __name__ == "__main__":
    path = build_library(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(path)
