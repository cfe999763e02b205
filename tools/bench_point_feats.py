"""Time the fused fine-pass point-feature sampler against the torch ops it replaces (fwd + bwd per scene).

LaRa's training size: V = 4 source views, n = 262 144 masked points, 512 x 512 images.  The renderings are handed
over as render_scene_views hands them over (channel-last views of planar buffers).  Both arms run in this call and
alternate; their outputs are compared at the same size.  The card name and power limit are read in the same call.

Prints the times and the agreement, then one JSON line.

    python tools/bench_point_feats.py [--reps 5] [--iters 50]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import rel_err  # noqa: E402
from lara_b200.point_feats import sample_point_feats  # noqa: E402
from test_point_feats import make_case, point_feats_torch  # noqa: E402
from timing import alternate, card, cuda_ms, summary  # noqa: E402


def restated_coords(points, w2c, ixt, H, W):
    """[V,n,2] grid_sample source coordinates (ix, iy) along the restatement's own chain of fp32 operations."""
    cam = points.reshape(1, -1, 3) @ w2c[:, :3, :3].permute(0, 2, 1) + w2c[:, :3, 3][:, None]
    cam = cam @ ixt.permute(0, 2, 1)
    wh = torch.tensor([W, H], device=points.device)
    g = (cam[..., :2] / cam[..., -1:] + 0.5) / wh * 2 - 1.0
    return ((g + 1) * wh - 1) / 2


def near_jump(coords, H, W, eps=1e-3):
    """[V,n] bool: a coordinate of the point that reaches the image lies within eps px of a pixel-centre line, where
    the point gradient jumps; the agreement of the point gradients is reported over the other points."""
    size = torch.tensor([W, H], dtype=coords.dtype, device=coords.device)
    c = coords.double()
    reaches = torch.isfinite(c) & (c > -1 - eps) & (c < size + eps)
    return (reaches & ((c - c.round()).abs() <= eps)).any(-1)


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

    for _ in range(10):
        for fn in arms.values():
            step(fn)
    times = alternate(arms, args.reps, lambda fn: 1e3 * cuda_ms(lambda: step(fn), args.iters))
    c = card()
    print(f"card: {c['name']}, power limit {c['power_limit']}")
    print(f"V={V} n={n} {H}x{W}, fwd+bwd per scene, {args.reps} alternating reps of {args.iters} steps (CUDA events)")
    res = {"card": c, "V": V, "n": n, "H": H, "W": W, "iters": args.iters}
    for name, ts in times.items():
        t = summary(ts)
        res[name] = {"fwd_bwd_us": t}
        print(f"  {name:24s} median {t['median']:9.1f} us   min {t['min']:9.1f}   max {t['max']:9.1f}")
    print("agreement (max |fused - torch| / max |torch|):")
    for k, v in agree.items():
        print(f"  {k:28s} {v:.2e}")
    res["agreement"] = agree
    print(json.dumps(res))


if __name__ == "__main__":
    main()
