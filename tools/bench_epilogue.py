"""Time the fused render_img epilogue against the torch ops it replaces (fwd + bwd, one view).

The two arms alternate within each of --repeats repeats of --iters calls, once timed with CUDA events and once with the
host clock.  Prints one line per arm and one JSON line with the card's name and power limit.

    python tools/bench_epilogue.py [SIZE=512] [--iters 100] [--repeats 5]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from timing import alternate, card, cuda_ms, host_ms, summary  # noqa: E402  (tools/ is on sys.path as a script)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("size", type=int, nargs="?", default=512, help="image height and width")
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    from lara_b200.epilogue import render_img_epilogue
    from oracle.torch_restatements import render_img_epilogue_torch
    from test_epilogue import _inputs

    dev = torch.device("cuda:0")
    H = W = a.size
    color, allmap, rays, vm = _inputs(H, W, 1, dev)
    allmap[1].clamp_(min=0.05)
    w = {k: torch.randn(s, device=dev) for k, s in (("image", (H, W, 3)), ("depth", (H, W, 1)), ("acc_map", (H, W)),
                                                    ("rend_normal", (H, W, 3)), ("depth_normal", (H, W, 3)),
                                                    ("rend_dist", (H, W)))}

    def step_of(fn):
        def step():
            c = color.clone().requires_grad_(True)
            am = allmap.clone().requires_grad_(True)
            out = fn(c, am, rays, vm, 0.0)
            torch.autograd.backward([out[k] for k in w], [w[k] for k in w])
        return step

    arms = {"torch ops (reference)": step_of(render_img_epilogue_torch), "fused kernel": step_of(render_img_epilogue)}
    for _ in range(10):
        for step in arms.values():
            step()
    gpu = alternate(arms, a.repeats, lambda step: 1e3 * cuda_ms(step, a.iters))
    wall = alternate(arms, a.repeats, lambda step: 1e3 * host_ms(lambda: [step() for _ in range(a.iters)]) / a.iters)
    res = {"card": card(), "H": H, "W": W, "iters": a.iters}
    for name in arms:
        res[name] = {"gpu_us_per_view": summary(gpu[name]), "wall_us_per_view": summary(wall[name])}
        print(f"{name:24s} {H}x{W}: {res[name]['gpu_us_per_view']['median']:8.1f} us/view GPU, "
              f"{res[name]['wall_us_per_view']['median']:8.1f} us/view wall")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
