"""Time the fused fine-pass point-feature sampler against the torch ops it replaces (fwd + bwd per scene).

LaRa's training size: V = 4 source views, n = 262 144 masked points, 512 x 512 images.  The renderings are handed
over as render_scene_views hands them over (channel-last views of planar buffers).  Both arms run in this call and
alternate; their outputs are compared at the same size.  The card name and power limit are read in the same call.

    python tools/bench_point_feats.py [--reps 5] [--iters 50]
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import rel_err  # noqa: E402
from lara_b200.point_feats import sample_point_feats  # noqa: E402
from test_point_feats import make_case, near_jump, point_feats_torch, restated_coords  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=4)
    ap.add_argument("--points", type=int, default=262144)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_point_feats: no CUDA device")
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    V, n, H = args.views, args.points, args.size
    W = H
    points, img_ref, rend, w2c, ixt = make_case(V, H, W, n, n, coarse=8)
    points, img_ref, w2c, ixt = points.to(dev), img_ref.to(dev), w2c.to(dev), ixt.to(dev)
    planar = {"image": rend["image"].permute(0, 3, 1, 2).contiguous().to(dev), "acc_map": rend["acc_map"].to(dev),
              "depth": rend["depth"].permute(0, 3, 1, 2).contiguous().to(dev)}
    leaves = [points.clone().requires_grad_(True)] + [t.clone().requires_grad_(True) for t in planar.values()]
    up = torch.randn((V, 8, n), generator=torch.Generator().manual_seed(1)).to(dev)

    def step(fn):
        pts, image, acc, depth = leaves
        r = {"image": image.permute(0, 2, 3, 1), "acc_map": acc, "depth": depth.permute(0, 2, 3, 1)}
        out = fn(pts, img_ref, r, w2c, ixt)
        return out.detach(), torch.autograd.grad(out, leaves, up)

    arms = {"torch ops (reference)": point_feats_torch, "fused kernels": sample_point_feats}
    res = {k: step(fn) for k, fn in arms.items()}
    (f1, g1), (f2, g2) = res["fused kernels"], res["torch ops (reference)"]
    keep = ~near_jump(restated_coords(points, w2c, ixt, H, W), H, W).any(0)
    agree = {"feats(max over channels)": max(rel_err(f1[:, c].cpu().numpy(), f2[:, c].cpu().numpy()) for c in range(8)),
             "g_points(kept %.2f%%)" % (100 * float(keep.float().mean())): rel_err(g1[0][keep].cpu().numpy(), g2[0][keep].cpu().numpy())}
    agree.update({f"g_{k}": rel_err(a.cpu().numpy(), b.cpu().numpy()) for k, a, b in zip(planar, g1[1:], g2[1:])})
    del res, f1, f2, g1, g2

    times = {k: [] for k in arms}
    for _ in range(10):
        for fn in arms.values():
            step(fn)
    torch.cuda.synchronize()
    for _ in range(args.reps):
        for name, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                step(fn)
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.iters * 1e3)
    print(f"card: {card}")
    print(f"V={V} n={n} {H}x{W}, fwd+bwd per scene, {args.reps} alternating reps of {args.iters} steps (CUDA events)")
    for name, ts in times.items():
        ts = sorted(ts)
        print(f"  {name:24s} median {ts[len(ts) // 2]:9.1f} us   min {ts[0]:9.1f}   max {ts[-1]:9.1f}")
    print("agreement (max |fused - torch| / max |torch|):")
    for k, v in agree.items():
        print(f"  {k:28s} {v:.2e}")


if __name__ == "__main__":
    main()
