"""LaRa's training loss for every scene of a batch (DESIGN §3.27): the per-scene recipe against ``Losses``.

At LaRa's size (B = 3 scenes, 8 target views of 512^2, coarse and fine pass, iter > 1000 so every term is on) the two
arms compute the loss and its backward to the planar render buffers, [B,V,3,H,W] leaves as the batch renders return:

* ``recipe``: INTEGRATION.md's former per-scene loop, ``scene_loss(out_i, tar_rgb[i], iter, batch_scenes=B,
  ms_ssim=True)`` per scene and pass, summed;
* ``losses``: ``lara_b200.loss.Losses()(batch, {**out_b, **out_fine_b}, iter)``.

The arms alternate over --repeats; each repeat times one forward + backward on the host clock around a device
synchronise.  In the same run: kernel launches per step from ``torch.profiler`` (a profiled window of its own, after
the timed one), the peak-allocation increase of one step, and the card's name and power limit.  Prints one JSON line.

    python tools/bench_batch_loss.py [--repeats 15]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from timing import alternate, card, host_ms, peak_mib, summary  # noqa: E402  (tools/ is on sys.path as a script)

B, V, H, W, ITER = 3, 8, 512, 512, 5000
GRAD_KEYS = ("image", "image_fine", "rend_normal", "depth_normal", "rend_dist")


def setup(dev):
    """Planar leaves [B,V,C,H,W] / [B,V,H,W], the [B,V,H,W,C] views of them the renders return, and tar_rgb."""
    g = torch.Generator(device=dev).manual_seed(3)
    tar = torch.rand(B, V, H, W, 3, generator=g, device=dev)
    leaves, views = {}, {}
    for k in ("image", "image_fine", "rend_normal", "depth_normal"):
        base = tar.permute(0, 1, 4, 2, 3) if k.startswith("image") else 0.5
        t = (0.8 * base + 0.2 * torch.rand(B, V, 3, H, W, generator=g, device=dev)).contiguous()
        leaves[k] = t.requires_grad_(True)
        views[k] = t.permute(0, 1, 3, 4, 2)
    for k in ("rend_dist", "acc_map", "acc_map_fine"):
        leaves[k] = (torch.rand(B, V, H, W, generator=g, device=dev) * 0.01).requires_grad_(k == "rend_dist")
        views[k] = leaves[k]
    return leaves, views, tar


def recipe(views, tar):
    from lara_b200.loss import scene_loss
    loss = 0
    for i in range(B):
        for prex in ("", "_fine"):
            out = {k: v[i] for k, v in views.items() if k.endswith("_fine") == (prex == "_fine")}
            loss_i, _ = scene_loss(out, tar[i], ITER, batch_scenes=B, prex=prex, ms_ssim=True)
            loss = loss + loss_i
    return loss


def step(arm, leaves, views, tar):
    from lara_b200.loss import Losses
    for k in GRAD_KEYS:
        leaves[k].grad = None
    loss = recipe(views, tar) if arm == "recipe" else Losses()({"tar_rgb": tar}, views, ITER)[0]
    loss.backward()
    return loss


def launches(fn, steps=3) -> float:
    """Kernel launches per call of ``fn`` in a torch.profiler window of ``steps`` calls."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    n = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
            and "memcpy" not in e.name.lower() and "memset" not in e.name.lower())
    return n / steps


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=15)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    leaves, views, tar = setup(dev)
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit']}", flush=True)
    res = {"card": info, "B": B, "V": V, "H": H, "W": W, "iter": ITER}
    arms = {name: (lambda name=name: step(name, leaves, views, tar)) for name in ("recipe", "losses")}
    for fn in arms.values():               # warm-up of every shape the timed window uses
        fn()
    # the two arms' losses and image gradients side by side (a different grouping of the same sums)
    la = float(arms["recipe"]())
    ga = leaves["image"].grad.clone()
    lb = float(arms["losses"]())
    gb = leaves["image"].grad
    res["agree"] = {"loss_rel_diff": abs(la - lb) / abs(la),
                    "g_image_rel_diff": float((ga - gb).abs().max() / ga.abs().max())}
    samples = alternate(arms, args.repeats, host_ms)
    res["step_ms"] = {k: summary(v) for k, v in samples.items()}
    res["kernel_launches_per_step"] = {k: launches(fn) for k, fn in arms.items()}
    res["peak_mib"] = {k: peak_mib(fn) for k, fn in arms.items()}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
