"""The coarse pass's feature-volume lifting per step (DESIGN §3.17): forward + backward of ``build_feat_vol``, the
view-embedding concatenation and ``VolTransformer.forward``'s blocks at LaRa's size (B = 3 scenes, V = 4 source views,
ViT-B/16 tokens on 512^2 images: C = 768 on a 32 x 32 map, R = 16, E = 32, n_group = 16), with C = 384 (ViT-S) as a
second point.

Three arms, alternating in one process after a warm-up: the fused op in the condition layout
(``FeatVolume.cond_tokens``), and LaRa's torch path (``oracle.feat_volume_torch``: build_feat_vol + cat + blocks, LaRa's
op sequence) in fp32 and under bf16 autocast.  Each is timed with CUDA events; the median and range over --repeats are
printed, with the peak-memory increase of one forward + backward.  The HBM floor is computed from shapes: the reads and
writes of the inputs, of y (the modulated token map, written once and read once) and of the output in the forward, and
of dL/dout, dL/dy (written and read), the token map and dL/dimg_feats in the backward, at 3.35 TB/s.  Prints the card's
name and power limit, then one JSON line.

    python tools/bench_feat_volume.py [--repeats 7] [--iters 10]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from timing import alternate, card, cuda_ms, peak_mib, summary  # noqa: E402  (tools/ is on sys.path as a script)

B, V, HW, IMG, R, E, NG = 3, 4, 32, 512, 16, 32, 16
HBM_BYTES_PER_S = 3.35e12


def floors_us(C: int) -> dict:
    T = B * V * HW * HW
    out = B * V * R ** 3 * (C + E)
    fwd = 4 * (T * C + T * 6 + 2 * T * C + out)          # x, rays, y written and read, output
    bwd = 4 * (out + 2 * T * C + T * C + T * C)          # dL/dout, dL/dy written and read, x, dL/dx
    return {"fwd_mb": fwd / 1e6, "bwd_mb": bwd / 1e6, "fwd_us": fwd / HBM_BYTES_PER_S * 1e6,
            "bwd_us": bwd / HBM_BYTES_PER_S * 1e6}


def run(C: int, repeats: int, iters: int) -> dict:
    from lara_b200.feat_volume import FeatVolume
    from oracle.feat_volume_torch import build_feat_vol_torch, cond_tokens_torch
    from test_feat_volume import make_case      # tests/ is on sys.path (below)
    dev = torch.device("cuda:0")
    img_feats, rays, w2c, ixt, params, ve = make_case(B, V, C, HW, HW, IMG, IMG, R, E, 0)
    fv = FeatVolume(C, E, R).to(dev)
    with torch.no_grad():
        for p, v in zip((fv.dir_norm.norm.weight, fv.dir_norm.norm.bias, fv.dir_norm.mlp[1].weight,
                         fv.dir_norm.mlp[1].bias), params):
            p.copy_(v)
        fv.view_embed.copy_(ve)
    x = img_feats.to(dev).requires_grad_(True)
    rays, w2c, ixt = rays.to(dev), w2c.to(dev), ixt.to(dev)
    up = torch.randn((B * NG ** 3, V * (R // NG) ** 3, C + E), device=dev)
    tparams = (fv.dir_norm.norm.weight, fv.dir_norm.norm.bias, fv.dir_norm.mlp[1].weight, fv.dir_norm.mlp[1].bias)

    def fused():
        fv.cond_tokens(x, rays, w2c, ixt, (IMG, IMG), NG).backward(up)

    def torch_path():
        vol = build_feat_vol_torch(x, rays, w2c, ixt, (IMG, IMG), fv.volume_grid, tparams)
        return cond_tokens_torch(vol, fv.view_embed, NG)

    def fp32():
        torch_path().backward(up)

    def bf16():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = torch_path()
        out.backward(up)

    arms = {"fused": fused, "torch_fp32": fp32, "torch_bf16_autocast": bf16}

    def clear():
        for t in [x, *fv.parameters()]:
            t.grad = None

    peak, failed = {}, {}
    for name, fn in list(arms.items()):
        try:
            fn()                                   # one call first: an arm that cannot run at this size is reported
        except RuntimeError as ex:
            failed[name] = str(ex).strip().splitlines()[0]
            del arms[name]
            clear()
            continue
        clear()
        for _ in range(2):                         # warm-up (and the first-call allocations)
            fn()
            clear()
        peak[name] = peak_mib(fn)
        clear()
    times = alternate(arms, repeats, lambda fn: 1e3 * cuda_ms(lambda: (fn(), clear()), iters))
    fl = floors_us(C)
    floor = fl["fwd_us"] + fl["bwd_us"]
    print(f"B={B} V={V} C={C} tokens {HW}x{HW} image {IMG}^2 R={R} E={E} n_group={NG}; HBM floor fwd "
          f"{fl['fwd_mb']:.0f} MB {fl['fwd_us']:.0f} us, bwd {fl['bwd_mb']:.0f} MB {fl['bwd_us']:.0f} us")
    res = {"C": C, "floor": {k: round(v, 1) for k, v in fl.items()}}
    for name, ts in times.items():
        t = summary(ts)
        print(f"  {name:22s} fwd+bwd {t['median']:9.1f} us (range {t['min']:.1f} - {t['max']:.1f})  "
              f"peak +{peak[name]:8.1f} MB  HBM-floor share {floor / t['median']:.2f}")
        res[name] = {"fwd_bwd_us": t, "peak_increase_mb": round(peak[name], 1),
                     "floor_share": round(floor / t["median"], 3)}
    for name, msg in failed.items():
        print(f"  {name:22s} fails at this size: {msg}")
        res[name] = {"error": msg}
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10, help="forward + backward calls per timed repeat")
    args = ap.parse_args()
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    c = card()
    print(f"card: {c['name']}, power limit {c['power_limit']}")
    res = {"card": c, "points": [run(C, args.repeats, args.iters) for C in (768, 384)]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
