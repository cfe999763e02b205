"""LaRa's volume transformer per step (DESIGN §3.19): forward + backward of the 12-layer ``VolTransformer`` at LaRa's
size (B = 3 scenes, C = 256, H = 16, R = 32, n_groups = [16], V = 4 views of C = 768 + 32 features on a 16^3 volume,
so each group's condition is [4, 800]; out_dim 80).

Four arms, alternating in one process after a warm-up: LaRa's VolTransformer (``oracle.vol_transformer_torch``, LaRa's
op sequence, bit-identical to LaRa's module on the CPU) and the drop-in (``lara_b200.vol_transformer``), each in fp32 and
under bf16 autocast, with torch's default TF32 settings.  Each is timed with CUDA events; the median and range over
--repeats are printed, with the peak-memory increase of one forward + backward.  Then, in separate runs, a
``torch.profiler`` split of one forward + backward of each arm into GEMM / convolution kernels, torch's SDPA kernels
and everything else
(with the largest other kernels and every copy or layout-transpose kernel), and whether each arm runs under
``torch.use_deterministic_algorithms(True)``.  Prints the card's name and power limit, then one JSON line.

    python tools/bench_vol_transformer.py [--repeats 5] [--iters 3] [--layers 12]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from timing import alternate, card, cuda_ms, peak_mib, summary  # noqa: E402  (tools/ is on sys.path as a script)

B, V, C, CC, H, R, RC, NG, OUT = 3, 4, 256, 800, 16, 32, 16, [16], 80
ATTN = ("fmha", "sdpa", "attention")          # torch's SDPA kernels (LaRa's attention core), before DENSE
DENSE = ("gemm", "xmma", "cutlass", "conv", "cudnn", "fprop", "dgrad", "wgrad", "implicit", "sm90", "cublas", "nvjet",
         "splitkreduce")
COPY = ("copy", "transpose", "nchwtonhwc", "nhwctonchw", "memcpy", "unfold", "im2col", "col2im", "cat")


def setup(layers: int):
    from lara_b200.vol_transformer import VolTransformer
    from oracle.vol_transformer_torch import vol_transformer_torch
    from test_vol_transformer import transformer_params
    dev = torch.device("cuda:0")
    p = {k: v.to(dev) for k, v in transformer_params(C, CC, R, OUT, layers, 1).items()}
    feats = torch.randn((B, V, CC, RC, RC, RC), device=dev).requires_grad_(True)
    up = torch.randn((B, 2 * R, 2 * R, 2 * R, OUT), device=dev)
    vt = VolTransformer(C, CC, NG, R, 2 * R, OUT, layers, H).to(dev)
    vt.load_state_dict(p, strict=True)
    lp = {k: v.clone().requires_grad_(True) for k, v in p.items()}

    def lara(bf16):
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=bf16):
            out = vol_transformer_torch(feats, lp, NG, H, R)
        out.backward(up)

    def drop_in(bf16):
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=bf16):
            out = vt(feats)
        out.backward(up)

    def clear():
        feats.grad = None
        for t in list(vt.parameters()) + list(lp.values()):
            t.grad = None
    arms = {"lara_fp32": lambda: lara(False), "drop_in_fp32": lambda: drop_in(False),
            "lara_bf16_autocast": lambda: lara(True), "drop_in_bf16_autocast": lambda: drop_in(True)}
    return arms, clear


def profile_split(fn, clear) -> dict:
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], record_shapes=True) as prof:
        fn()
        torch.cuda.synchronize()
    clear()
    kernels = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            k = kernels.setdefault(ev.name, [0.0, 0])
            k[0] += ev.device_time / 1e3
            k[1] += 1
    attn = sum(t for n, (t, _) in kernels.items() if any(s in n.lower() for s in ATTN))
    dense = sum(t for n, (t, _) in kernels.items()
                if any(s in n.lower() for s in DENSE) and not any(s in n.lower() for s in ATTN))
    other = {n: v for n, v in kernels.items() if not any(s in n.lower() for s in DENSE + ATTN)}
    copies = {n[:90]: (round(t, 3), c) for n, (t, c) in kernels.items() if any(s in n.lower() for s in COPY)}
    # the copies torch issues (aten::copy_ under contiguous / clone / to / expand), by shape: a full-volume one moves
    # at least B R^3 C elements
    full = B * R ** 3 * C
    host_copies = {}
    for ev in prof.events():
        if ev.name == "aten::copy_" and ev.input_shapes and ev.input_shapes[0]:
            shape = tuple(ev.input_shapes[0])
            n = 1
            for s_ in shape:
                n *= s_
            key = f"{shape}{' full-volume' if n >= full else ''}"
            host_copies[key] = host_copies.get(key, 0) + 1
    top = sorted(other.items(), key=lambda kv: -kv[1][0])[:14]
    return {"dense_ms": round(dense, 2), "sdpa_ms": round(attn, 2), "other_ms": round(sum(t for t, _ in other.values()), 2),
            "top_other": [(n[:140], round(t, 3), c) for n, (t, c) in top], "copy_kernels": copies,
            "aten_copies": host_copies,
            "top_dense": [(n[:140], round(t, 3), c) for n, (t, c) in sorted(kernels.items(), key=lambda kv: -kv[1][0])
                          if any(s in n.lower() for s in DENSE + ATTN)][:6]}


def deterministic_ok(fn, clear) -> str:
    was = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        fn()
        torch.cuda.synchronize()
        return "runs"
    except RuntimeError as ex:
        return "raises: " + str(ex).strip().splitlines()[0][:160]
    finally:
        torch.use_deterministic_algorithms(was)
        clear()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3, help="forward + backward calls per timed repeat")
    ap.add_argument("--layers", type=int, default=12)
    args = ap.parse_args()
    c = card()
    print(f"card: {c['name']}, power limit {c['power_limit']}")
    arms, clear = setup(args.layers)
    peak = {}
    for name, fn in arms.items():
        for _ in range(2):                         # warm-up (and the first-call allocations)
            fn()
            clear()
        peak[name] = peak_mib(fn)
        clear()
    times = alternate(arms, args.repeats, lambda fn: cuda_ms(lambda: (fn(), clear()), args.iters))
    print(f"B={B} V={V} C={C} cond {CC} H={H} R={R} n_groups={NG} layers={args.layers} out {OUT}")
    res = {"card": c, "layers": args.layers}
    for name, ts in times.items():
        t = summary(ts)
        print(f"  {name:24s} fwd+bwd {t['median']:8.2f} ms (range {t['min']:.2f} - {t['max']:.2f})  "
              f"peak +{peak[name]:8.1f} MB")
        res[name] = {"fwd_bwd_ms": t, "peak_increase_mb": round(peak[name], 1)}
    for name, fn in arms.items():
        split = profile_split(fn, clear)
        res[name]["profile"] = split
        print(f"  {name:24s} profiler: GEMM/conv {split['dense_ms']:.2f} ms, SDPA {split['sdpa_ms']:.2f} ms, "
              f"other {split['other_ms']:.2f} ms")
        for n, t, cnt in split["top_other"]:
            print(f"      {t:8.3f} ms  x{cnt:<4d} {n}")
        for n, t, cnt in split["top_dense"]:
            print(f"      dense {t:8.3f} ms  x{cnt:<4d} {n}")
        print(f"      copy / transpose kernels: {split['copy_kernels']}")
        print(f"      aten::copy_ by destination shape: {split['aten_copies']}")
    for name in ("lara_fp32", "drop_in_fp32"):
        res[name]["deterministic_algorithms"] = deterministic_ok(arms[name], clear)
        print(f"  {name:24s} under torch.use_deterministic_algorithms(True): {res[name]['deterministic_algorithms']}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
