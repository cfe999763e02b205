#!/usr/bin/env python
"""Per-kernel device time (srf_profile_*, CUDA events around every launch) of the batched launch set.

    python tools/time_kernels.py [--P 131072] [--size 512] [--views 8] [--steps 5]

Prints one JSON line: us per VIEW per kernel (launch time / views per launch) and the step time."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from lara_b200 import _lib, rasterizer as R, scene as S, sharded  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--P", type=int, default=131072)
ap.add_argument("--size", type=int, default=512)
ap.add_argument("--views", type=int, default=8)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--sh", type=int, default=1)
args = ap.parse_args()

dev = torch.device("cuda:0")
sc = S.scene(args.P, 0, sh_degree=args.sh)
cams = S.cameras(args.views, args.size, args.size, 0)
gc, ga = S.upstream_grads(args.size, args.size, 0, lara_like=True)
params = {k: sc[k].to(dev) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
bg = torch.ones(3)
sets = [S.settings_for(c, bg, args.sh, dev, R.GaussianRasterizationSettings) for c in cams]
G = (gc.to(dev).expand(args.views, -1, -1, -1).contiguous(), ga.to(dev).expand(args.views, -1, -1, -1).contiguous())
grads = sharded.GradBuffer(args.P, int(params["shs"].shape[1]), dev)
packed = R.pack_cameras(sets, dev)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def step():
    grads.zero_()
    sharded.render_views(params, sets, None, grads=grads, upstream_stacked=G, cams=packed)


def measure():
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    _lib.profile_begin()
    for _ in range(args.steps):
        flush.zero_()
        step()
    torch.cuda.synchronize()
    k = _lib.profile_end()
    st = [torch.cuda.Event(enable_timing=True) for _ in range(2 * args.steps)]
    for i in range(args.steps):
        flush.zero_()
        st[2 * i].record(); step(); st[2 * i + 1].record()
    torch.cuda.synchronize()
    ms = sum(st[2 * i].elapsed_time(st[2 * i + 1]) for i in range(args.steps)) / args.steps
    out = {"P": args.P, "size": args.size, "views": args.views,
           "us_per_view": {n: round(t[0] * 1e3 / max(t[1], 1) / args.views, 2) for n, t in k.items()},
           "launches": {n: t[1] for n, t in k.items()},
           "step_ms": round(ms, 4), "views_per_s": round(args.views / ms * 1e3, 1)}
    print(json.dumps(out), flush=True)


measure()
