"""The benchmark tools' timing harness (tools/timing.py), no GPU: the order in which ``alternate`` runs the arms,
``summary`` on even and odd counts, ``card``'s fallback without nvidia-smi, and that every measuring function refuses
to run without CUDA."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import timing  # noqa: E402


def test_alternate_runs_the_arms_in_turn_inside_each_repeat():
    calls = []
    arms = {"a": lambda: "a", "b": lambda: "b", "c": lambda: "c"}

    def measure(fn):
        calls.append(fn())
        return len(calls)

    samples = timing.alternate(arms, 3, measure)
    assert calls == ["a", "b", "c"] * 3
    assert samples == {"a": [1, 4, 7], "b": [2, 5, 8], "c": [3, 6, 9]}
    assert list(samples) == ["a", "b", "c"]


def test_summary_on_odd_and_even_counts():
    assert timing.summary([5.0, 1.0, 3.0]) == {"median": 3.0, "min": 1.0, "max": 5.0, "n": 3}
    assert timing.summary([4.0, 1.0, 8.0, 2.0]) == {"median": 3.0, "min": 1.0, "max": 8.0, "n": 4}
    assert timing.summary([2.5]) == {"median": 2.5, "min": 2.5, "max": 2.5, "n": 1}


def test_card_falls_back_without_nvidia_smi(monkeypatch):
    def missing(*args, **kwargs):
        raise FileNotFoundError("nvidia-smi")

    monkeypatch.setattr(timing.subprocess, "run", missing)
    monkeypatch.setattr(torch.cuda, "get_device_name", lambda *a: "Some GPU")
    assert timing.card() == {"name": "Some GPU", "power_limit": "unknown"}


def test_card_reads_name_and_power_limit(monkeypatch):
    class Done:
        stdout = "NVIDIA H100 80GB HBM3, 700.00 W\n"

    seen = []
    monkeypatch.setattr(timing.subprocess, "run", lambda cmd, **kw: seen.append(cmd) or Done())
    assert timing.card() == {"name": "NVIDIA H100 80GB HBM3", "power_limit": "700.00 W"}
    assert seen == [["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"]]


@pytest.mark.parametrize("call", [lambda f: timing.cuda_ms(f, 3), timing.host_ms, timing.peak_mib],
                         ids=["cuda_ms", "host_ms", "peak_mib"])
def test_measuring_functions_raise_without_cuda(monkeypatch, call):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    ran = []
    with pytest.raises(RuntimeError, match="no CUDA device"):
        call(lambda: ran.append(1))
    assert ran == []
