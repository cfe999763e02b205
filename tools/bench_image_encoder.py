"""LaRa's image encoder per step (DESIGN §3.25): ViT-B/16 (``vit_base_patch16_224.dino``) on 12 images of 512 x 512
(LaRa's B = 3 scenes x 4 source views), forward + backward and forward only.

Arms, alternating in one process after a warm-up: the fused encoder (``lara_b200.image_encoder.DinoEncoder``) and the
restatement of timm's forward (``oracle.vit_torch``), each in fp32 with torch's defaults, in fp32 under LaRa's
``torch.set_float32_matmul_precision('medium')``, and under bf16 autocast (LaRa trains with ``bf16-mixed``).  Each is
timed with CUDA events; the median and range over --repeats are printed, with the peak-memory increase of one call.
Then, in separate runs, a ``torch.profiler`` split of one forward + backward into GEMM, SDPA and other kernels, and the
SDPA kernels the fused arms run under ``torch.use_deterministic_algorithms(True)``.  Prints
the card's name and power limit, then one JSON line.

    python tools/bench_image_encoder.py [--repeats 5] [--iters 3]
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

N, H, W, C, HEADS = 12, 512, 512, 768, 12
ATTN = ("fmha", "sdpa", "attention", "flash")
DENSE = ("gemm", "xmma", "cutlass", "sm90", "cublas", "nvjet", "splitkreduce")
PRECISION = {"fp32": ("highest", False), "fp32_medium": ("medium", False), "bf16_autocast": ("highest", True)}


def setup():
    from lara_b200.image_encoder import DinoEncoder
    from oracle.vit_torch import vit_forward
    from test_image_encoder import vit_params
    dev = torch.device("cuda:0")
    p = {k: v.to(dev) for k, v in vit_params(C, 12, 1).items()}
    img = torch.rand((N, 3, H, W), device=dev)
    up = torch.randn((N, (H // 16) * (W // 16), C), device=dev)
    enc = DinoEncoder("vit_base_patch16_224.dino", is_train=True).to(dev)
    enc.model.load_state_dict(p, strict=True)
    lp = {k: v.clone().requires_grad_(True) for k, v in p.items()}

    def run(fused, prec, backward):
        precision, bf16 = PRECISION[prec]
        torch.set_float32_matmul_precision(precision)
        try:
            with torch.set_grad_enabled(backward), torch.autocast("cuda", dtype=torch.bfloat16, enabled=bf16):
                out = enc(img) if fused else vit_forward(img, lp, HEADS)
            if backward:
                out.backward(up)
        finally:
            torch.set_float32_matmul_precision("highest")

    def clear():
        for t in list(enc.parameters()) + list(lp.values()):
            t.grad = None
    arms = {}
    for mode, bwd in (("fwd_bwd", True), ("fwd", False)):
        for prec in PRECISION:
            for name, fused in (("restatement", False), ("fused", True)):
                arms[f"{name}_{prec}_{mode}"] = (lambda f=fused, p_=prec, b=bwd: run(f, p_, b))
    return arms, clear


def profile_split(fn, clear) -> dict:
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    clear()
    kernels = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            k = kernels.setdefault(ev.name, [0.0, 0])
            k[0] += ev.device_time / 1e3
            k[1] += 1
    is_attn = lambda n: any(s in n.lower() for s in ATTN)                     # noqa: E731
    is_dense = lambda n: any(s in n.lower() for s in DENSE) and not is_attn(n)  # noqa: E731
    attn = {n: v for n, v in kernels.items() if is_attn(n)}
    other = {n: v for n, v in kernels.items() if not is_attn(n) and not is_dense(n)}
    return {"gemm_ms": round(sum(t for n, (t, _) in kernels.items() if is_dense(n)), 2),
            "sdpa_ms": round(sum(t for t, _ in attn.values()), 2),
            "other_ms": round(sum(t for t, _ in other.values()), 2),
            "sdpa_kernels": [(n[:120], round(t, 3), c) for n, (t, c) in sorted(attn.items(), key=lambda kv: -kv[1][0])],
            "top_other": [(n[:120], round(t, 3), c) for n, (t, c) in sorted(other.items(), key=lambda kv: -kv[1][0])[:10]]}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3, help="calls per timed repeat")
    args = ap.parse_args()
    c = card()
    print(f"card: {c['name']}, power limit {c['power_limit']}")
    arms, clear = setup()
    peak = {}
    for name, fn in arms.items():
        for _ in range(2):                         # warm-up (and the first-call allocations)
            fn()
            clear()
        peak[name] = peak_mib(fn)
        clear()
    times = alternate(arms, args.repeats, lambda fn: cuda_ms(lambda: (fn(), clear()), args.iters))
    print(f"N={N} images of {H}x{W}, ViT-B/16 (C={C}, {HEADS} heads, 12 blocks)")
    res = {"card": c}
    for name, ts in times.items():
        t = summary(ts)
        print(f"  {name:36s} {t['median']:8.2f} ms (range {t['min']:.2f} - {t['max']:.2f})  peak +{peak[name]:8.1f} MB")
        res[name] = {"ms": t, "peak_increase_mb": round(peak[name], 1)}
    for name, fn in arms.items():
        if not name.endswith("fwd_bwd"):
            continue
        split = profile_split(fn, clear)
        res[name]["profile"] = split
        print(f"  {name:36s} profiler: GEMM {split['gemm_ms']:.2f} ms, SDPA {split['sdpa_ms']:.2f} ms, "
              f"other {split['other_ms']:.2f} ms")
        for n, t, cnt in split["sdpa_kernels"]:
            print(f"      sdpa {t:8.3f} ms  x{cnt:<4d} {n}")
        for n, t, cnt in split["top_other"]:
            print(f"      {t:8.3f} ms  x{cnt:<4d} {n}")
    was = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        for name in ("fused_fp32_fwd_bwd", "fused_bf16_autocast_fwd_bwd"):
            split = profile_split(arms[name], clear)
            res[name]["sdpa_kernels_deterministic"] = split["sdpa_kernels"]
            print(f"  {name:36s} under torch.use_deterministic_algorithms(True): SDPA {split['sdpa_ms']:.2f} ms")
            for n, t, cnt in split["sdpa_kernels"]:
                print(f"      sdpa {t:8.3f} ms  x{cnt:<4d} {n}")
    finally:
        torch.use_deterministic_algorithms(was)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
