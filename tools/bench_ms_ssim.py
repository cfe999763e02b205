"""Time the fused MS-SSIM kernels against the library's op sequence (ms_ssim_torch), forward + backward.

Two workloads at LaRa's training size (configs/base.yaml: 3 scenes x 8 target views of 512 x 512):
  module : MS_SSIM on [3, 3, 512, 4096] passed as LaRa passes it, a channel-last view (output['image'].permute(0,3,1,2));
  scenes : 3 x scene_loss(ms_ssim=True) on V = 8 planar 512^2 views, against ms_ssim_torch on each scene's
           torch.cat of the views (the MS-SSIM term alone in both arms).
Both arms of a workload alternate in this call, every shape is warmed up first, the profiler is off, and the outputs
are compared at the same size.  The card name and power limit are read in the same call.

Prints the times and the agreement, then one JSON line.

    python tools/bench_ms_ssim.py [--reps 5] [--iters 50]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import rel_err  # noqa: E402
from lara_b200.loss import scene_loss  # noqa: E402
from lara_b200.ssim import MS_SSIM  # noqa: E402
from test_ms_ssim import ms_ssim_torch, smooth_pair  # noqa: E402
from timing import alternate, card, cuda_ms, summary  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=3)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ms_ssim: no CUDA device")
    dev = torch.device("cuda:0")
    B, V, H = args.scenes, args.views, args.size
    X, Y = smooth_pair(B * V, 3, H, H, 7, dtype=torch.float32)
    # planar per-scene views [B][V,3,H,W] as the fused epilogue writes them; targets [B][V,H,W,3] as the batch holds them
    views = X.reshape(B, V, 3, H, H).to(dev)
    tars = Y.reshape(B, V, 3, H, H).permute(0, 1, 3, 4, 2).contiguous().to(dev)
    # LaRa's concatenated image [B,H,V*W,3] and its channel-last view
    img_cl = views.permute(0, 3, 1, 4, 2).reshape(B, H, V * H, 3).contiguous()
    tar_cl = tars.permute(0, 2, 1, 3, 4).reshape(B, H, V * H, 3).contiguous()
    mod = MS_SSIM(data_range=1.0, size_average=True, channel=3)

    def module_arm(fn):
        def step():
            x = img_cl.detach().requires_grad_(True)
            v = fn(x.permute(0, 3, 1, 2), tar_cl.permute(0, 3, 1, 2))
            (0.5 * (1 - v)).backward()
            return v.detach(), x.grad
        return step

    def scenes_fused():
        vs, gs = [], []
        for b in range(B):
            x = views[b].detach().requires_grad_(True)
            loss, st = scene_loss({"image": x.permute(0, 2, 3, 1)}, tars[b], 10, batch_scenes=B, ms_ssim=True)
            loss.backward()
            vs.append(st["ssim"])
            gs.append(x.grad)
        return sum(vs), torch.stack(gs)

    def scenes_torch():
        vs, gs = [], []
        for b in range(B):
            x = views[b].detach().requires_grad_(True)
            cat = torch.cat(list(x), dim=-1).unsqueeze(0)
            tcat = torch.cat(list(tars[b].permute(0, 3, 1, 2)), dim=-1).unsqueeze(0)
            v = ms_ssim_torch(cat, tcat, data_range=1.0)
            ((0.5 / B) * (1 - v)).backward()
            vs.append(v.detach() / B)
            gs.append(x.grad)
        return sum(vs), torch.stack(gs)

    # scenes_torch leaves out the MSE term that scene_loss always has; its gradient is subtracted for the comparison
    def mse_grad():
        gs = []
        for b in range(B):
            x = views[b].detach().requires_grad_(True)
            loss, _ = scene_loss({"image": x.permute(0, 2, 3, 1)}, tars[b], 10, batch_scenes=B)
            loss.backward()
            gs.append(x.grad)
        return torch.stack(gs)

    workloads = {
        f"module [{B},3,{H},{V * H}] channel-last": {"library op sequence (ms_ssim_torch)": module_arm(ms_ssim_torch),
                                                     "fused kernels (MS_SSIM)": module_arm(mod)},
        f"{B} x scene_loss(ms_ssim=True), V={V} planar {H}^2": {"library op sequence (ms_ssim_torch)": scenes_torch,
                                                               "fused kernels (scene_loss)": scenes_fused},
    }
    agree = {}
    for wname, arms in workloads.items():
        (vt, gt), (vf, gf) = [fn() for fn in arms.values()]
        if "scene_loss" in wname:
            gf = gf - mse_grad()
        agree[wname] = (abs(float(vf) - float(vt)), rel_err(gf.cpu().numpy(), gt.cpu().numpy()), float(vt))
    for arms in workloads.values():
        for _ in range(5):
            for fn in arms.values():
                fn()
    calls = {(w, a): fn for w, arms in workloads.items() for a, fn in arms.items()}
    times = alternate(calls, args.reps, lambda fn: 1e3 * cuda_ms(fn, args.iters))
    c = card()
    print(f"card: {c['name']}, power limit {c['power_limit']}")
    print(f"fwd+bwd of the MS-SSIM term, {args.reps} alternating reps of {args.iters} steps (CUDA events), us per step")
    res = {"card": c, "iters": args.iters}
    for wname, arms in workloads.items():
        print(f"{wname}:")
        d, g, v = agree[wname]
        res[wname] = {"agreement": {"value": v, "abs_value_diff": d, "grad_rel_err": g}}
        for name in arms:
            t = summary(times[(wname, name)])
            res[wname][name] = {"fwd_bwd_us": t}
            print(f"  {name:40s} median {t['median']:10.1f}   min {t['min']:10.1f}   max {t['max']:10.1f}")
        print(f"  agreement: value {v:.7f}, |fused - torch| {d:.2e}; dL/dimage max|fused - torch| / max|torch| {g:.2e}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
