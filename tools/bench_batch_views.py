"""What rendering the B scenes of a batch in one launch set saves (DESIGN §3.21): LaRa's per-scene render loop
(``render_scene_views`` then ``render_subset_views`` for each scene) against ``render_batch_views`` then
``render_batch_subset_views``, alternated in one process.

One step of each arm: the coarse render of every scene with a fixed random linear loss of its six maps, the fine
subset render (LaRa's opacity cut and training half-drop as masks, new SH coefficients) with the same kind of loss, and
one backward through both to the [B,P,...] leaves.  The first step of each arm checks that their outputs agree bit
for bit.  Per arm: the median and range over --rounds alternations of the mean of --iters steps, each timed with CUDA
events; then, in separate steps, the torch.profiler per-kernel device time and the peak memory of one step.
Prints the card's name and power limit, then one JSON line per arm and a summary line.

    python tools/bench_batch_views.py [--B 3] [--P 524288] [--views 8] [--size 512] [--iters 5] [--rounds 7]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from collections import defaultdict

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from timing import alternate, card, cuda_ms, peak_mib, summary  # noqa: E402  (tools/ is on sys.path as a script)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=3)
    ap.add_argument("--P", type=int, default=524288)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_batch_views needs a CUDA device")
    from lara_b200 import rasterizer as R, scene as S
    from lara_b200.multiview import (OUT_KEYS, render_batch_subset_views, render_batch_views, render_scene_views,
                                     render_subset_views)

    dev = torch.device("cuda:0")
    B, P, V, H = args.B, args.P, args.views, args.size
    print(json.dumps({"card": card(), "B": B, "P": P, "views": V, "size": H}), flush=True)
    params, settings, rays, masks, fine = [], [], [], [], []
    g = torch.Generator(device=dev).manual_seed(1)
    for b in range(B):
        sc = S.scene(P, b)
        params.append([t.to(dev) for t in (sc["means3D"], sc["shs"], torch.logit(sc["opacities"]),
                                           torch.log(sc["scales"]), sc["rotations"] * 1.7)])
        cams = S.cameras(V, H, H, b, fov=0.7 + 0.05 * b)
        settings.append([S.settings_for(c, torch.ones(3), sc["sh_degree"], dev, R.GaussianRasterizationSettings)
                         for c in cams])
        rays.append(torch.stack([torch.cat([c.c2w[:3, 3].expand(H, H, 3), torch.randn(H, H, 3)], -1) for c in cams]).to(dev))
        lara = torch.sigmoid(params[-1][2]).view(-1) > 0.005
        masks.append(lara & (torch.rand((P,), generator=g, device=dev) < 0.5))
        fine.append(torch.randn((int(masks[-1].sum()),) + tuple(sc["shs"].shape[1:]), generator=g, device=dev) * 0.6)
    leaves = [torch.stack([p[k] for p in params]).contiguous().requires_grad_(True) for k in range(5)]
    rays_b, masks_b = torch.stack(rays).contiguous(), torch.stack(masks)
    fine_b = torch.cat(fine).requires_grad_(True)
    fine_s = [f.detach().clone().requires_grad_(True) for f in fine]
    w = {k: None for k in OUT_KEYS}

    def weights(out, suffix):
        for k in OUT_KEYS:
            if w[k] is None:
                w[k] = torch.randn(out[k + suffix].shape, generator=g, device=dev)
        return w

    def loop_step():
        loss, images = 0.0, []
        for b in range(B):
            one = [t[b] for t in leaves]
            co = render_scene_views(*one, settings[b], rays=rays[b], raw_activations=True, keep_binning=True)
            fo = render_subset_views(co["binning"], masks[b], fine_s[b])
            ww = weights({k: torch.empty((B,) + tuple(co[k].shape)) for k in OUT_KEYS}, "")
            loss = loss + sum((co[k] * ww[k][b]).sum() + (fo[k + "_fine"] * ww[k][b]).sum() for k in OUT_KEYS)
            images.append((co["image"].detach(), fo["image_fine"].detach()))
        loss.backward()
        return images

    def batch_step():
        co = render_batch_views(*leaves, settings, rays=rays_b, raw_activations=True, keep_binning=True)
        fo = render_batch_subset_views(co["binning"], masks_b, fine_b)
        ww = weights(co, "")
        loss = sum((co[k] * ww[k]).sum() + (fo[k + "_fine"] * ww[k]).sum() for k in OUT_KEYS)
        loss.backward()
        return [(co["image"][b].detach(), fo["image_fine"][b].detach()) for b in range(B)]

    arms = {"loop": loop_step, "batch": batch_step}
    a, bt = loop_step(), batch_step()
    same = all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(a, bt))
    for _ in range(2):
        for fn in arms.values():
            fn()

    def clear_then(fn):
        for t in leaves + [fine_b] + fine_s:
            t.grad = None
        fn()

    times = alternate(arms, args.rounds, lambda fn: cuda_ms(lambda: clear_then(fn), args.iters))
    res = {}
    for name, fn in arms.items():
        peak = peak_mib(fn)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        kern = defaultdict(float)
        for ev in prof.key_averages():
            if ev.device_type.name == "CUDA" and ev.self_device_time_total > 0:
                kern[ev.key[:60]] += ev.self_device_time_total / 1000.0
        top = dict(sorted(kern.items(), key=lambda kv: -kv[1])[:14])
        res[name] = {"ms": summary(times[name]),
                     "kernel_ms_total": round(sum(kern.values()), 3), "peak_MB": round(peak, 1),
                     "kernels_ms": {k: round(v, 3) for k, v in top.items()}}
        print(json.dumps({"arm": name, **res[name]}), flush=True)
    loop_ms, batch_ms = res["loop"]["ms"]["median"], res["batch"]["ms"]["median"]
    print(json.dumps({"bit_identical": same, "speedup": loop_ms / batch_ms, "saved_ms": loop_ms - batch_ms}),
          flush=True)


if __name__ == "__main__":
    main()
