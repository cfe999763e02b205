#!/usr/bin/env python
"""Per-kernel device time (srf_profile_*, CUDA events around every launch) of the batched launch set.

    python tools/time_kernels.py [--P 131072] [--size 512] [--views 8] [--steps 5]

Prints one JSON line: the card's name and power limit, us per VIEW per kernel (launch time / views per launch) and the
step time, each step timed alone with CUDA events after a 256 MB write that evicts L2."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from timing import card, cuda_ms, summary  # noqa: E402  (tools/ is on sys.path when run as a script)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=131072)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--sh", type=int, default=1)
    args = ap.parse_args()
    from lara_b200 import _lib, rasterizer as R, scene as S, sharded

    dev = torch.device("cuda:0")
    sc = S.scene(args.P, 0, sh_degree=args.sh)
    cams = S.cameras(args.views, args.size, args.size, 0)
    gc, ga = S.upstream_grads(args.size, args.size, 0, lara_like=True)
    params = {k: sc[k].to(dev) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    sets = [S.settings_for(c, torch.ones(3), args.sh, dev, R.GaussianRasterizationSettings) for c in cams]
    G = (gc.to(dev).expand(args.views, -1, -1, -1).contiguous(), ga.to(dev).expand(args.views, -1, -1, -1).contiguous())
    grads = sharded.GradBuffer(args.P, int(params["shs"].shape[1]), dev)
    packed = R.pack_cameras(sets, dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def step():
        grads.zero_()
        sharded.render_views(params, sets, None, grads=grads, upstream_stacked=G, cams=packed)

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    _lib.profile_begin()
    for _ in range(args.steps):
        flush.zero_()
        step()
    torch.cuda.synchronize()
    k = _lib.profile_end()
    ms = []
    for _ in range(args.steps):
        flush.zero_()
        ms.append(cuda_ms(step, 1))
    t = summary(ms)
    out = {"card": card(), "P": args.P, "size": args.size, "views": args.views,
           "us_per_view": {n: round(v[0] * 1e3 / max(v[1], 1) / args.views, 2) for n, v in k.items()},
           "launches": {n: v[1] for n, v in k.items()},
           "step_ms": t, "views_per_s": round(args.views / t["median"] * 1e3, 1)}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
