"""What rendering LaRa's fine pass from the coarse pass's binning saves (DESIGN §3.18): the gathered path (four masked
gathers, ``render_scene_views`` on the gathered Gaussians, and the gathers' backward) against ``render_subset_views`` on
the coarse call's ``keep_binning`` state, alternated in one process.

Both arms render the same masked Gaussians with the same new SH coefficients into the same six maps, and the first
call of each checks that they agree bit for bit.  Per mask: the median over --rounds alternations of the mean of --iters
calls, each timed with CUDA events from the mask to completion (fwd+bwd: the fine render, a fixed random linear loss of
its six maps and its backward to the coarse leaves; fwd: under ``torch.no_grad``), then the per-kernel device time per
call from ``srf_profile_*`` (what the library's own kernels do not cover -- gathers, the subset kernels, the epilogue,
allocations -- is ``other``).  The coarse render runs once, untimed, with raw activations as in LaRa.  Masks: LaRa's
opacity cut ``sigmoid(opacity) > 0.005`` and the training half-drop on top of it.  Prints the card's name and power
limit, then one JSON line per (mask, mode).

    python tools/bench_subset_render.py [--P 524288] [--views 8] [--size 512] [--iters 10] [--rounds 5]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from timing import alternate, card, cuda_ms, summary  # noqa: E402  (tools/ is on sys.path when run as a script)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=524288)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_subset_render needs a CUDA device")
    from lara_b200 import _lib, rasterizer as R, scene as S
    from lara_b200.multiview import OUT_KEYS, render_scene_views, render_subset_views

    dev = torch.device("cuda:0")
    P, V, H = args.P, args.views, args.size
    print(json.dumps({"card": card(), "P": P, "views": V, "size": H}), flush=True)
    sc = S.scene(P, 0)
    cams = S.cameras(V, H, H, 0)
    settings = [S.settings_for(c, torch.ones(3), sc["sh_degree"], dev, R.GaussianRasterizationSettings) for c in cams]
    rays = torch.stack([torch.cat([c.c2w[:3, 3].expand(H, H, 3), torch.randn(H, H, 3)], -1) for c in cams]).to(dev)
    leaves = [t.to(dev).contiguous().requires_grad_(True) for t in
              (sc["means3D"], sc["shs"], torch.logit(sc["opacities"]), torch.log(sc["scales"]), sc["rotations"] * 1.7)]
    c, shs, o, s, r = leaves
    out = render_scene_views(c, shs, o, s, r, settings, rays=rays, raw_activations=True, keep_binning=True)
    binning = out["binning"]
    g = torch.Generator(device=dev).manual_seed(1)
    lara = torch.sigmoid(o.detach()).view(-1) > 0.005
    masks = {"lara": lara, "half_drop": lara & (torch.rand(P, generator=g, device=dev) < 0.5)}
    shs_all = torch.randn(shs.shape, generator=g, device=dev) * 0.5
    weights = {k: torch.randn(out[k].shape, generator=g, device=dev) for k in OUT_KEYS}

    def fine(arm, mask, shs_f):
        if arm == "subset":
            return render_subset_views(binning, mask, shs_f)
        return render_scene_views(c[mask], shs_f, o[mask], s[mask], r[mask], settings, rays=rays, raw_activations=True,
                                  prex="_fine")

    def call(arm, mask, shs_f, bwd):
        if not bwd:
            with torch.no_grad():
                return fine(arm, mask, shs_f)
        f = fine(arm, mask, shs_f)
        loss = sum((f[k + "_fine"] * weights[k]).sum() for k in OUT_KEYS)
        torch.autograd.grad(loss, [c, o, s, r, shs_f])
        return f

    for name, mask in masks.items():
        n = int(mask.sum())
        shs_f = shs_all[mask].contiguous().requires_grad_(True)
        with torch.no_grad():
            a, b = call("subset", mask, shs_f, False), call("gathered", mask, shs_f, False)
        same = all(torch.equal(a[k + "_fine"], b[k + "_fine"]) for k in OUT_KEYS + ("radii",))
        for bwd in (True, False):
            for arm in ("gathered", "subset", "gathered", "subset"):       # warm-up
                call(arm, mask, shs_f, bwd)
            arms = {arm: (lambda arm=arm: call(arm, mask, shs_f, bwd)) for arm in ("gathered", "subset")}
            t = {k: summary(v) for k, v in alternate(arms, args.rounds, lambda fn: cuda_ms(fn, args.iters)).items()}
            split = {}
            for arm in ("gathered", "subset"):
                torch.cuda.synchronize()
                _lib.profile_begin()
                for _ in range(args.iters):
                    call(arm, mask, shs_f, bwd)
                torch.cuda.synchronize()
                k = _lib.profile_end()
                per = {kk: round(ms / args.iters, 4) for kk, (ms, cnt) in k.items() if cnt}
                per["other"] = round(t[arm]["median"] - sum(per.values()), 4)
                split[arm] = per
            rec = {"mask": name, "n": n, "fraction": round(n / P, 4), "mode": "fwd+bwd" if bwd else "fwd",
                   "bit_identical_forward": same,
                   "gathered_ms": t["gathered"], "subset_ms": t["subset"], "kernels_ms": split,
                   "speedup": round(t["gathered"]["median"] / t["subset"]["median"], 3)}
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
