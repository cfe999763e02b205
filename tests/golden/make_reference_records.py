"""Record what the UNMODIFIED reference computes for the tests that compare against it
(tests/golden/reference/<module>.npz), so that those tests run without the reference.

Each listed test module has a ``record_reference(ref, dev)`` that runs the reference side of its
comparisons and returns ``{case: {field: value}}``; ``dev`` is ``cuda:0`` for the modules that drive the
reference's CUDA rasterizer (built into oracle/_ref by oracle/build_ref.py) and ``cpu`` for those that
run LaRa's own torch code on the CPU (``ref`` is then the path of the LaRa checkout).

    python tests/golden/make_reference_records.py gpu OUT_DIR     # on an H100, with oracle/_ref built
    python tests/golden/make_reference_records.py cpu OUT_DIR LARA_CHECKOUT
    cp OUT_DIR/*.npz tests/golden/reference/
"""
from __future__ import annotations

import importlib
import os
import sys

import numpy as np

TESTS = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROOT = os.path.dirname(TESTS)
sys.path[:0] = [ROOT, TESTS]

from helpers import flatten_record  # noqa: E402

GPU_MODULES = ["test_gpu_parity", "test_gpu_headline", "test_gpu_edges", "test_gpu_readback", "test_epilogue",
               "test_renderer_callsite"]
CPU_MODULES = ["test_epilogue_cpu", "test_decoder_layout", "test_loss"]


PART_BYTES = 900_000     # a module's cases are split over <module>.npz, <module>.1.npz, ... of at most this much data


def save(out_dir, name, recs):
    parts, part, size = [], {}, 0
    for case, r in recs.items():
        flat = {f"{case}/{k}": np.asarray(v) for k, v in flatten_record(r).items()}
        nbytes = sum(a.nbytes for a in flat.values())
        if part and size + nbytes > PART_BYTES:
            parts.append(part)
            part, size = {}, 0
        part.update(flat)
        size += nbytes
    parts.append(part)
    for i, p in enumerate(parts):
        np.savez_compressed(os.path.join(out_dir, name + (f".{i}" if i else "") + ".npz"), **p)
    print(name, len(recs), "cases in", len(parts), "file(s)", flush=True)


def main(kind, out_dir, lara=None):
    os.makedirs(out_dir, exist_ok=True)
    if kind == "gpu":
        import torch
        from oracle import ref as REF
        ref, dev = REF.load(), torch.device("cuda:0")
        for name in GPU_MODULES:
            save(out_dir, name, importlib.import_module(name).record_reference(ref, dev))
    else:
        for name in CPU_MODULES:
            mod, fn = name.removesuffix("_cpu"), "record_reference_cpu" if name.endswith("_cpu") else "record_reference"
            save(out_dir, name, getattr(importlib.import_module(mod), fn)(lara, "cpu"))


if __name__ == "__main__":
    main(*sys.argv[1:])
