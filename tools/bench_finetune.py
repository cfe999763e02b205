"""Time the per-scene refinement loop on one GPU (DESIGN §3.24).

Workload: LaRa's evaluation size, 4 source views of 512^2 and ``scene(P)`` (degree-1 SH, M = 4) at P = 131 072 and
262 144 Gaussians, LaRa's learning rates; the targets are the scene's own renders and the refined copy starts from a
seeded perturbation of it.  Arms, alternating, ``--steps`` refinement steps each, medians over ``--reps``:

  A  ``finetune_scene``: ``Renderer.render_views``, ``scene_loss(..., ms_ssim=True)``, one ``GaussianAdam`` launch;
  B  the same render and loss, ``torch.optim.Adam(foreach=False)`` over get_params' six leaves and a ``torch.cat`` of
     f_dc and f_rest each step (isolates the optimiser);
  C  a per-view ``Renderer.render_img`` loop stacked with ``torch.stack``, the SH tensor rebuilt with ``torch.cat``,
     the same loss and Adam as B: how the loop reads when written against LaRa's own renderer interface.

Also the Adam kernel alone (CUDA events over ``--kernel-iters`` launches) and its bytes/s against the H100 SXM's
3.35 TB/s; the card's name and power limit are read in the same run.  One JSON line per P.

    python tools/bench_finetune.py [--P 131072 262144] [--steps 20] [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from lara_b200 import finetune as F  # noqa: E402
from lara_b200.loss import scene_loss  # noqa: E402
from lara_b200.renderer import Renderer  # noqa: E402
from lara_b200.scene import PathCamera, cameras, scene  # noqa: E402
from timing import alternate, card, cuda_ms, host_ms, summary  # noqa: E402  (tools/ is on sys.path as a script)

LRS = dict(position_lr=0.000016, feature_lr=0.0025, opacity_lr=0.05, scaling_lr=0.005, rotation_lr=0.001)
HBM_BYTES_PER_S = 3.35e12


def make_case(P, V, H, dev, seed=0):
    sc = scene(P, seed)
    raw = [sc["means3D"], sc["shs"], torch.logit(sc["opacities"]), torch.log(sc["scales"]), sc["rotations"]]
    cams = cameras(V, H, H, seed)
    c2w = torch.stack([c.c2w for c in cams])
    sample = {"tar_c2w": c2w[None].to(dev), "fovx": torch.tensor([0.75], device=dev),
              "fovy": torch.tensor([0.75], device=dev), "near_far": torch.tensor([[0.5, 2.5]], device=dev),
              "bg_color": torch.ones((1, V, 3), device=dev),
              "tar_rays": torch.stack([PathCamera(c2w[j], H, H, 0.75).get_rays()[0] for j in range(V)])[None].to(dev)}
    renderer = Renderer(sh_degree=sc["sh_degree"])
    mask = torch.ones(P, dtype=torch.bool, device=dev)
    gt = [t.to(dev) for t in raw]
    with torch.no_grad():
        out = renderer.render_views(F.sample_cameras({**sample, "tar_rgb": torch.empty(1, V, H, H, 3, device=dev)}, range(V)),
                                    sample["tar_rays"][0], *gt, dev, bg_colors=sample["bg_color"][0])
    sample["tar_rgb"] = out["image"].contiguous()[None]
    g = torch.Generator().manual_seed(100 + seed)
    start = [(t.cpu() + k * torch.randn(t.shape, generator=g)).to(dev)
             for t, k in zip(raw, (0.001, 0.1, 0.5, 0.1, 0.02))]
    return renderer, sample, (*start, mask)


def torch_adam_loop(renderer, gs, sample, V, steps, per_view):
    """Arms B (per_view=False) and C (per_view=True)."""
    c, s, o, sc, r, mask = gs
    dev = c.device
    leaves = [c.clone(), s[:, :1].clone(), s[:, 1:].clone(), o[mask].clone(), sc[mask].clone(), r[mask].clone()]
    for t in leaves:
        t.requires_grad_(True)
    lrs = F.group_lrs(**LRS)
    opt = torch.optim.Adam([{"params": [t], "lr": lr, "name": k} for t, lr, k in zip(leaves, lrs, F.GROUPS)],
                           betas=(0.9, 0.999), eps=1e-15, foreach=False)
    cams = F.sample_cameras(sample, range(V))
    rays, tar, bg = (sample[k][0, :V] for k in ("tar_rays", "tar_rgb", "bg_color"))
    losses = torch.empty(steps, device=dev)
    for i in range(steps):
        shs = torch.cat(leaves[1:3], 1)
        if per_view:
            frames = []
            for j, cam in enumerate(cams):
                renderer.set_bg_color(bg[j])
                frames.append(renderer.render_img(cam, rays[j], leaves[0], shs, *leaves[3:], dev))
            out = {k: torch.stack([f[k] for f in frames]) for k in ("image", "rend_normal", "depth_normal",
                                                                       "rend_dist", "acc_map")}
        else:
            out = renderer.render_views(cams, rays, leaves[0], shs, *leaves[3:], dev, bg_colors=bg)
        loss, _ = scene_loss(out, tar, 1001, batch_scenes=1, ms_ssim=True)
        loss.backward()
        losses[i] = loss.detach()
        opt.step()
        opt.zero_grad()
    return losses


def kernel_time(P, M, dev, iters):
    g = torch.Generator().manual_seed(1)
    ts = [torch.randn(s, generator=g).to(dev).requires_grad_(True) for s in ((P, 3), (P, M, 3), (P, 1), (P, 2), (P, 4))]
    opt = F.GaussianAdam(*ts, **LRS)
    for t in ts:
        t.grad = torch.randn_like(t)
    for _ in range(10):
        opt.step()
    ms = cuda_ms(opt.step, iters)
    nbytes = 32 * P * (10 + 3 * M)         # reads param, grad, two moments; writes param, two moments, zeroed grad
    return ms, nbytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, nargs="+", default=[131072, 262144])
    ap.add_argument("--views", type=int, default=4)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--kernel-iters", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_finetune: needs a CUDA device")
    dev = torch.device("cuda:0")
    gpu = card()
    V = args.views
    for P in args.P:
        renderer, sample, gs = make_case(P, V, args.size, dev)
        arms = {"A_fused": lambda: F.finetune_scene(renderer, gs, sample, V, args.steps, **LRS)[1],
                "B_torch_adam": lambda: torch_adam_loop(renderer, gs, sample, V, args.steps, False),
                "C_render_img": lambda: torch_adam_loop(renderer, gs, sample, V, args.steps, True)}
        for fn in arms.values():           # warm every shape
            fn()
        times = alternate(arms, args.reps, host_ms)
        ms, nbytes = kernel_time(P, int(gs[1].shape[1]), dev, args.kernel_iters)
        res = {"card": gpu, "P": P, "views": V, "size": args.size, "steps": args.steps, "reps": args.reps}
        for k, v in times.items():
            t = summary(v)
            res[f"{k}_steps_per_s"] = round(1e3 * args.steps / t["median"], 2)
            res[f"{k}_steps_per_s_range"] = [round(1e3 * args.steps / t["max"], 2),
                                             round(1e3 * args.steps / t["min"], 2)]
        res["adam_kernel_ms"] = round(ms, 4)
        res["adam_kernel_TBps"] = round(nbytes / (ms * 1e-3) / 1e12, 3)
        res["adam_kernel_share_of_3.35TBps"] = round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
