"""Per-kernel device time of the two per-Gaussian kernels, preprocess_fwd and preprocess_bwd (srf_profile_*), on the
paths that launch them, and optionally the same against a second build of the library in one process.

    python tools/time_preprocess.py [--against OTHER.so] [--steps 10] [--rounds 7] [--out FILE.json]

Paths, all at 512² with 8 views per scene and LaRa's SH degree 1 unless named otherwise:
  s1_acc      one scene, accumulating backward: ``sharded.render_views`` (bench.py's ``value``), P = 131 072
  s1_131k     one scene, overwriting backward: ``render_scene_views`` + backward, P = 131 072
  s1_524k     the same at P = 524 288
  s3_524k     three scenes in one launch set: ``render_batch_views`` + backward, P = 524 288 per scene
  s1_131k_sh3 ``s1_131k`` at SH degree 3 (M = 16), the backward's general-M path

``--against`` loads a second ``libsurfel_b200.so`` of the same ABI (built from another revision) and alternates the
two libraries round by round, so the spread of each over the rounds is measured next to their difference.  Before
timing, each path runs once per library with ``torch.use_deterministic_algorithms(True)`` and the outputs (colour,
aux maps, radii) and gradients are compared bit for bit.  Prints the card's name and power limit, then one JSON line
per (path, library) with the median, minimum and maximum over the rounds of the us per launch of each kernel.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from timing import alternate, card, summary  # noqa: E402

KERNELS = ("preprocess_fwd", "preprocess_bwd")


def bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def make_paths(dev, size, views):
    from lara_b200 import rasterizer as R, scene as S, sharded
    from lara_b200.multiview import render_batch_views, render_scene_views

    def settings(b, fov=0.75, sh=1):
        return [S.settings_for(c, torch.ones(3), sh, dev, R.GaussianRasterizationSettings)
                for c in S.cameras(views, size, size, b, fov=fov)]

    def leaves(P, b, sh):
        sc = S.scene(P, b, sh_degree=sh)
        return [t.to(dev) for t in (sc["means3D"], sc["shs"], torch.logit(sc["opacities"]), torch.log(sc["scales"]),
                                    sc["rotations"] * 1.7)]

    def weighted_loss(out, g):
        return sum((t * w).sum() for t, w in zip(out, g))

    def acc_path(P):
        sc = S.scene(P, 0)
        params = {k: sc[k].to(dev) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
        sets = settings(0)
        gc, ga = S.upstream_grads(size, size, 0, lara_like=True)
        G = (gc.to(dev).expand(views, -1, -1, -1).contiguous(), ga.to(dev).expand(views, -1, -1, -1).contiguous())
        grads = sharded.GradBuffer(P, int(params["shs"].shape[1]), dev)
        cams = R.pack_cameras(sets, dev)

        def step():
            grads.zero_()
            outs, _ = sharded.render_views(params, sets, None, grads=grads, upstream_stacked=G, cams=cams)
            return [t for o in outs for t in o] + [grads.flat]
        return step

    def scene_path(P, B, sh=1):
        ls = [leaves(P, b, sh) for b in range(B)]
        sets = [settings(b, 0.7 + 0.05 * b, sh) for b in range(B)]
        x = [torch.stack([l[k] for l in ls]).contiguous().requires_grad_(True) for k in range(5)]
        rays = torch.randn((B, views, size, size, 6), generator=torch.Generator().manual_seed(B)).to(dev)
        g = None

        def step():
            nonlocal g
            for t in x:
                t.grad = None
            if B == 1:
                out = render_scene_views(*[t[0] for t in x], sets[0], rays=rays[0], raw_activations=True)
            else:
                out = render_batch_views(*x, sets, rays=rays, raw_activations=True)
            maps = [out[k] for k in sorted(out) if k != "radii"]
            if g is None:
                gen = torch.Generator(device=dev).manual_seed(7)
                g = [torch.randn(t.shape, generator=gen, device=dev) for t in maps]
            weighted_loss(maps, g).backward()
            return [t.detach() for t in maps] + [out["radii"]] + [t.grad for t in x]
        return step

    return {"s1_acc": acc_path(131072), "s1_131k": scene_path(131072, 1), "s1_524k": scene_path(524288, 1),
            "s3_524k": scene_path(524288, 3), "s1_131k_sh3": scene_path(131072, 1, sh=3)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--against", default=None, help="a second libsurfel_b200.so to alternate with the in-tree one")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--out", default=None, help="also write the results to this JSON file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_preprocess needs a CUDA device")
    from lara_b200 import _lib

    libs = {"tree": _lib.load()}
    if args.against:
        libs["against"] = _lib.load(os.path.abspath(args.against))
    dev = torch.device("cuda:0")
    print(json.dumps({"card": card(), "libs": {k: getattr(v, "_name", "") for k, v in libs.items()}}), flush=True)
    paths = make_paths(dev, args.size, args.views)

    def use(name):
        _lib._lib = libs[name]

    parity = {}
    for pname, step in paths.items():
        torch.use_deterministic_algorithms(True)
        res = {}
        for lname in libs:
            use(lname)
            res[lname] = [t.clone() for t in step()]
        torch.use_deterministic_algorithms(False)
        if len(libs) > 1:
            a, b = res["tree"], res["against"]
            parity[pname] = len(a) == len(b) and all(torch.equal(bits(x), bits(y)) for x, y in zip(a, b))
    if parity:
        print(json.dumps({"bit_identical": parity}), flush=True)

    def profiled(step, lname):
        """us per launch of each of KERNELS over --steps steps with library ``lname``."""
        use(lname)
        torch.cuda.synchronize()
        _lib.profile_begin()
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
        prof = _lib.profile_end()
        return {k: prof[k][0] * 1e3 / max(prof[k][1], 1) for k in KERNELS}

    results = []
    for pname, step in paths.items():
        for lname in libs:
            use(lname)
            for _ in range(3):
                step()
        times = alternate({l: l for l in libs}, args.rounds, lambda lname: profiled(step, lname))
        for lname in libs:
            row = {"path": pname, "lib": lname}
            for k in KERNELS:
                row[k + "_us"] = summary([t[k] for t in times[lname]])
            results.append(row)
            print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": card(), "bit_identical": parity, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
