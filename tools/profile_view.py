"""Run a few fwd+bwd views of one implementation and time them: device time (CUDA events) and wall time (host clock
from a synchronised device to a synchronised device), per view.  Prints one line and one JSON line with the card's
name and power limit.

    python tools/profile_view.py --impl mine|ref --P 131072 --size 512 --iters 5
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from timing import card, cuda_ms, host_ms  # noqa: E402  (tools/ is on sys.path when run as a script)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--impl", default="mine")
    ap.add_argument("--P", type=int, default=131072)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    from lara_b200 import rasterizer as R, scene as S
    from oracle import ref as REF

    dev = torch.device("cuda:0")
    mod = R if a.impl == "mine" else REF.load()
    sc = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in S.scene(a.P, 0).items()}
    cam = S.cameras(1, a.size, a.size, 0)[0]
    st = S.settings_for(cam, torch.ones(3), 1, dev, mod.GaussianRasterizationSettings)
    gc, ga = [t.to(dev) for t in S.upstream_grads(a.size, a.size, 0, lara_like=True)]
    leaves = {k: sc[k].clone().requires_grad_(True) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    m2d = torch.zeros_like(leaves["means3D"], requires_grad=True)

    def step():
        rast = mod.GaussianRasterizer(raster_settings=st)
        c, rd, am = rast(means3D=leaves["means3D"], means2D=m2d, shs=leaves["shs"], opacities=leaves["opacities"],
                         scales=leaves["scales"], rotations=leaves["rotations"])
        torch.autograd.backward((c, am), (gc, ga))

    for _ in range(a.warmup):
        step()
    gpu = cuda_ms(step, a.iters)
    wall = host_ms(lambda: [step() for _ in range(a.iters)]) / a.iters
    print(f"{a.impl} P={a.P} {a.size}^2: gpu {gpu:.3f} ms/view, wall {wall:.3f} ms/view")
    print(json.dumps({"card": card(), "impl": a.impl, "P": a.P, "size": a.size, "iters": a.iters,
                      "gpu_ms_per_view": gpu, "wall_ms_per_view": wall}))


if __name__ == "__main__":
    main()
