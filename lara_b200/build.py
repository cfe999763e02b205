"""In-tree build of the C-ABI library ``lara_b200/libsurfel_b200.so``.

Plain ``nvcc`` command lines (no torch, no setuptools): the library has no
dependency on libtorch -- it takes raw device pointers and a ``cudaStream_t``.
sm_90a only (H100): ``-gencode arch=compute_90a,code=sm_90a``, ``-lineinfo`` so ncu's
source page maps to the .cu files, nvcc's default ``-fmad=true`` and *no*
``--use_fast_math`` (the integer-critical float chains are pinned with explicit
intrinsics anyway, see csrc/surfel_common.cuh).

    python -m lara_b200.build          # build if sources are newer than the .so
    python -m lara_b200.build --force [--ptxas-info]     # registers / spills per kernel
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libsurfel_b200.so")
SOURCES = ["api.cu", "preprocess.cu", "binning.cu", "render_fwd.cu", "render_bwd.cu", "preprocess_bwd.cu", "epilogue.cu", "loss.cu", "decoder.cu", "point_feats.cu"]
HEADERS = ["surfel_common.cuh", "surfel_kernels.h", os.path.join("..", "..", "include", "surfel_rasterizer.h")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
]


def _nvcc() -> str:
    return os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def _newest_source_mtime() -> float:
    paths = [os.path.join(CSRC, s) for s in SOURCES] + [os.path.join(CSRC, h) for h in HEADERS]
    return max(os.path.getmtime(p) for p in paths)


def needs_build() -> bool:
    return (not os.path.isfile(LIB)) or os.path.getmtime(LIB) < _newest_source_mtime()


def build(force: bool = False, verbose: bool = True, ptxas_info: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    hdr_mtime = max(os.path.getmtime(os.path.join(CSRC, h)) for h in HEADERS)

    def compile_one(src: str) -> str:
        path = os.path.join(CSRC, src)
        obj = os.path.join(OBJ, src + ".o")
        if (not force and os.path.isfile(obj)
                and os.path.getmtime(obj) > max(os.path.getmtime(path), hdr_mtime)):
            return obj
        cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if ptxas_info else []) + ["-c", path, "-o", obj]
        if verbose:
            print("[lara_b200.build]", " ".join(cmd), flush=True)
        subprocess.run(cmd, check=True)
        return obj

    with ThreadPoolExecutor(max_workers=min(len(SOURCES), os.cpu_count() or 1)) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    cmd = [_nvcc(), "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"]
    if verbose:
        print("[lara_b200.build]", " ".join(cmd), flush=True)
    subprocess.run(cmd, check=True)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, ptxas_info="--ptxas-info" in sys.argv))
