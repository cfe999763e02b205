"""The one module the benchmark tools under tools/ measure with.

* :func:`card` -- the card's name and power limit, which belong beside every number measured on it;
* :func:`cuda_ms` -- device time per call from CUDA events around ``iters`` calls;
* :func:`host_ms` -- host clock around one call that starts and ends with a device synchronise;
* :func:`peak_mib` -- the increase of the peak allocation during one call;
* :func:`alternate` -- the arms of a comparison take turns inside each repeat, so drift on a shared machine lands on
  every arm alike;
* :func:`summary` -- median, min, max and count of a list of samples.

The measuring functions raise without CUDA: there is no CPU fallback for a time.
"""
from __future__ import annotations

import statistics
import subprocess
import time

import torch


def card() -> dict:
    """``{"name", "power_limit"}`` of the first card from the read-only ``nvidia-smi`` query, or torch's device name and
    ``"unknown"`` where that query is not available."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except Exception:                    # noqa: BLE001  (no nvidia-smi, or output of another form)
        name, power = torch.cuda.get_device_name(), "unknown"
    return {"name": name, "power_limit": power}


def _need_cuda() -> None:
    if not torch.cuda.is_available():
        raise RuntimeError("timing: no CUDA device; a time is only measured on the GPU")


def cuda_ms(fn, iters: int) -> float:
    """ms per call of ``fn``: CUDA events around ``iters`` calls, after a synchronise and read after another."""
    _need_cuda()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def host_ms(fn) -> float:
    """ms of one call of ``fn`` on the host clock, from a synchronised device to a synchronised device."""
    _need_cuda()
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def peak_mib(fn) -> float:
    """MiB by which the peak of ``torch.cuda.max_memory_allocated`` during one call of ``fn`` exceeds the allocation
    before it."""
    _need_cuda()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def alternate(arms: dict, repeats: int, measure) -> dict:
    """``{arm: [measure(fn) per repeat]}``; within each repeat every arm of ``arms`` (name -> callable) is measured
    once, in order."""
    samples = {name: [] for name in arms}
    for _ in range(repeats):
        for name, fn in arms.items():
            samples[name].append(measure(fn))
    return samples


def summary(samples) -> dict:
    """``{"median", "min", "max", "n"}`` of a non-empty list of samples."""
    return {"median": statistics.median(samples), "min": min(samples), "max": max(samples), "n": len(samples)}
