"""Build recipe for ``oracle/_ref`` -- TEST INFRASTRUCTURE ONLY, never shipped.

Compiles the *unmodified* reference rasterizer (LaRa's
``third_party/diff-surfel-rasterization``) from the LaRa checkout at ``REF_ROOT``
(``LARA_REFERENCE_ROOT`` overrides it) into ``oracle/_ref/diff_surfel_rasterization/``
so that

  * ``tests/golden/make_reference_records.py`` can record what the real reference
    computes for the GPU parity tests (they read the records, not this build), and
  * ``bench.py --impl reference`` can time the reference's own CUDA build.

Nothing under ``lara_b200/`` imports this.  ``oracle/_ref/`` is build output and
git-ignored.

The recipe is our own (plain nvcc / g++ command lines, no use of the
reference's setup.py or CMake).  One extra flag is needed with gcc-13:
``-include cstdint`` (``rasterizer_impl.h:24`` uses ``std::uintptr_t`` without
including it).  Device code is built for ``compute_90 / sm_90`` with nvcc's
default optimisation and *no* fast-math -- what the reference's own
``setup.py:22-30`` would produce with ``TORCH_CUDA_ARCH_LIST=9.0``.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = os.environ.get("LARA_REFERENCE_ROOT", "/root/reference")
DSR = os.path.join(REF_ROOT, "third_party", "diff-surfel-rasterization")
OUT = os.path.join(HERE, "_ref")
PKG = os.path.join(OUT, "diff_surfel_rasterization")
OBJ = os.path.join(OUT, "obj")

SOURCES = [
    "cuda_rasterizer/rasterizer_impl.cu",
    "cuda_rasterizer/forward.cu",
    "cuda_rasterizer/backward.cu",
    "rasterize_points.cu",
    "ext.cpp",
]


def reference_available() -> bool:
    return os.path.isfile(os.path.join(DSR, "ext.cpp"))


def built() -> bool:
    return os.path.isfile(os.path.join(PKG, "_C.so")) and os.path.isfile(
        os.path.join(PKG, "__init__.py"))


def _torch_flags():
    import torch
    from torch.utils import cpp_extension as ce
    inc = []
    for p in ce.include_paths("cuda"):
        inc += ["-isystem", p]
    inc += ["-isystem", sysconfig.get_paths()["include"]]
    libdir = os.path.join(os.path.dirname(torch.__file__), "lib")
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    defs = [
        "-DTORCH_API_INCLUDE_EXTENSION_H",
        "-DTORCH_EXTENSION_NAME=_C",
        f"-D_GLIBCXX_USE_CXX11_ABI={abi}",
    ]
    return inc, libdir, defs


def build(verbose: bool = True) -> str:
    """Compile the reference into oracle/_ref; returns the package directory."""
    if not reference_available():
        raise RuntimeError(f"reference sources not found under {DSR}")
    os.makedirs(PKG, exist_ok=True)
    os.makedirs(OBJ, exist_ok=True)
    inc, libdir, defs = _torch_flags()
    glm = os.path.join(DSR, "third_party", "glm")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

    def compile_one(src):
        path = os.path.join(DSR, src)
        obj = os.path.join(OBJ, src.replace("/", "_") + ".o")
        if os.path.exists(obj) and os.path.getmtime(obj) > os.path.getmtime(path):
            return obj
        if src.endswith(".cu"):
            cmd = [nvcc, "-c", path, "-o", obj, "-std=c++17",
                   "-gencode=arch=compute_90,code=sm_90",
                   "-D__CUDA_NO_HALF_OPERATORS__", "-D__CUDA_NO_HALF_CONVERSIONS__",
                   "-D__CUDA_NO_BFLOAT16_CONVERSIONS__", "-D__CUDA_NO_HALF2_OPERATORS__",
                   "--expt-relaxed-constexpr", "-include", "cstdint",
                   "--compiler-options", "-fPIC", "-w",
                   "-I", glm, "-I", DSR] + defs + inc
        else:
            cmd = ["g++", "-c", path, "-o", obj, "-std=c++17", "-O2", "-fPIC", "-w",
                   "-include", "cstdint", "-I", DSR] + defs + inc
        if verbose:
            print("[oracle/_ref]", " ".join(cmd[:6]), "...", flush=True)
        subprocess.run(cmd, check=True)
        return obj

    with ThreadPoolExecutor(max_workers=min(5, os.cpu_count() or 1)) as ex:
        objs = list(ex.map(compile_one, SOURCES))

    so = os.path.join(PKG, "_C.so")
    link = ["g++", "-shared", "-o", so] + objs + [
        f"-L{libdir}", "-L/usr/local/cuda/lib64",
        "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python",
        "-lcudart", f"-Wl,-rpath,{libdir}",
    ]
    subprocess.run(link, check=True)
    # The reference's Python surface (autograd.Function etc.), installed next to the
    # extension exactly as `pip install --target` would place it.  Install output only:
    # lives under the git-ignored oracle/_ref, never in history.
    shutil.copyfile(os.path.join(DSR, "diff_surfel_rasterization", "__init__.py"),
                    os.path.join(PKG, "__init__.py"))
    return PKG


if __name__ == "__main__":
    build()
    print("built", PKG)
