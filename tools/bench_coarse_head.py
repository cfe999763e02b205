"""The coarse-pass decoder head per step (DESIGN §3.20): ``mlp_coarse`` and the Gaussian layout at LaRa's size
(B = 3 scenes, 64^3 voxels, D = 80, K = 2, sh_dim 12: 786 432 rows, 1 572 864 Gaussians), with a fixed random upstream
gradient on the five outputs.

Four arms, alternating in one process after a warm-up:
  fused        ``CoarseHead.gaussians``;
  repo_fp32    torch's ``mlp_coarse`` + ``gaussians_from_decoder`` (the path before the fused head);
  lara_fp32    LaRa's ``Decoder.forward_coarse`` + ``Network.get_offseted_pt`` as written there (restated by
               ``oracle.coarse_head_torch``, bit-exact with it), plus the ``.contiguous()`` of sh and rotation that each
               rasterizer call performs;
  lara_bf16    the same under bf16 autocast (LaRa trains with ``precision="bf16-mixed"``), reported only.
Each arm is timed with CUDA events for forward + backward and for the forward alone under ``no_grad``; the median and
range over --repeats are printed, with the peak-memory increase of one forward + backward.  The floors from shapes
(HBM bytes at 3.35 TB/s, multiply-adds) and the card's name and power limit are printed, then one JSON line.

    python tools/bench_coarse_head.py [--repeats 7] [--iters 10]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from timing import alternate, card, cuda_ms, peak_mib, summary  # noqa: E402  (tools/ is on sys.path as a script)

B, R, D, K, SH = 3, 64, 80, 2, 12
OPACITY_SHIFT, SCALING_SHIFT, HALF_CELL = -2.1792, -4.2, 0.5 * 0.5 / 32


def floors():
    """HBM bytes and multiply-adds from shapes (fp32).  Forward: read feats, write the five outputs.  Backward: read
    feats and the five upstream gradients, write dL/dfeats.  Multiply-adds: the three layers forward, and forward
    again + two products per layer (dL/dinput, dL/dW) in the backward."""
    rows, O = B * R ** 3, K * (10 + SH)
    act, out = 4 * rows * D, 4 * rows * O
    fwd_bytes, bwd_bytes = act + out, act + out + act
    macs = rows * (D * D * 2 + D * O)
    return {"fwd_hbm_mb": fwd_bytes / 1e6, "bwd_hbm_mb": bwd_bytes / 1e6, "fwd_floor_us": fwd_bytes / 3.35e6,
            "bwd_floor_us": bwd_bytes / 3.35e6, "fwd_gmac": macs / 1e9, "fwd_bwd_gmac_recompute": 4 * macs / 1e9}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10, help="calls per timed repeat")
    args = ap.parse_args()
    from lara_b200 import CoarseHead
    from lara_b200.decoder_layout import gaussians_from_decoder
    from oracle.coarse_head_torch import coarse_head_torch
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    head = CoarseHead(D, SH, K).to(dev)
    feats = torch.randn((B, R, R, R, D), device=dev, generator=g).requires_grad_(True)
    gc = (torch.rand((1, R ** 3, 3), device=dev, generator=g) - 0.5) * 0.5
    G = R ** 3 * K
    ups = [torch.randn(s, device=dev, generator=g) for s in ((B, G, 3), (B, G, SH // 3, 3), (B, G, 2), (B, G, 4),
                                                              (B, G, 1))]

    def fused():
        return head.gaussians(feats, gc, OPACITY_SHIFT, SCALING_SHIFT, HALF_CELL)

    def repo():
        y = head.mlp_coarse(feats).float().reshape(B, R ** 3, -1)
        return gaussians_from_decoder(y, gc, K, SH, OPACITY_SHIFT, SCALING_SHIFT, HALF_CELL)

    def lara():
        c, sh, sc, rot, op = coarse_head_torch(feats, head._params(), K, SH, OPACITY_SHIFT, SCALING_SHIFT,
                                               gc, HALF_CELL)
        return c, sh.contiguous(), sc, rot.contiguous(), op

    def lara_bf16():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            return lara()

    arms = {"fused": fused, "repo_fp32": repo, "lara_fp32": lara, "lara_bf16": lara_bf16}

    def step(fn):
        torch.autograd.backward(fn(), ups)

    def forward(fn):
        with torch.no_grad():
            fn()

    def clear():
        for t in [feats, *head.parameters()]:
            t.grad = None

    peak = {}
    for name, fn in arms.items():
        for _ in range(2):                         # warm-up (and the first-call allocations)
            step(fn)
            forward(fn)
            clear()
        peak[name] = peak_mib(lambda: step(fn))
        clear()
    # each arm's forward + backward, then its forward alone; the arms alternate within each repeat
    calls = {(name, mode): (lambda run=run, fn=fn: (run(fn), clear()))
             for name, fn in arms.items() for mode, run in (("fwd_bwd", step), ("fwd", forward))}
    times = alternate(calls, args.repeats, lambda call: 1e3 * cuda_ms(call, args.iters))
    c = card()
    fl = floors()
    print(f"card: {c['name']}, power limit {c['power_limit']}; B={B} voxels={R}^3 D={D} K={K} sh_dim={SH}")
    print(f"  floors: HBM fwd {fl['fwd_hbm_mb']:.0f} MB = {fl['fwd_floor_us']:.0f} us, bwd {fl['bwd_hbm_mb']:.0f} MB = "
          f"{fl['bwd_floor_us']:.0f} us at 3.35 TB/s; {fl['fwd_gmac']:.1f} G multiply-adds forward, "
          f"{fl['fwd_bwd_gmac_recompute']:.1f} G forward + backward with the recompute")
    res = {"card": c, "B": B, "voxels": R ** 3, "D": D, "K": K, "sh_dim": SH, "floors": fl}
    for name in arms:
        r = {"peak_increase_mb": round(peak[name], 1)}
        line = f"  {name:10s}"
        for mode in ("fwd_bwd", "fwd"):
            t = summary(times[(name, mode)])
            r[mode + "_us"] = t
            line += f"  {mode} {t['median']:8.1f} us ({t['min']:.1f} - {t['max']:.1f})"
        print(line + f"  peak +{peak[name]:7.1f} MB")
        res[name] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
