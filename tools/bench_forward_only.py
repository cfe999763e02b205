"""What the forward-only path saves (DESIGN §3.14): the training forward (srf_scenes_forward with for_backward = 1, with
the contribution record and the image state the backward reads) against the forward-only one (for_backward = 0) on the
same inputs, alternated in one process.

Per point: the whole call (forward_views_raw, enqueue to completion) timed with CUDA events, the mean of --iters calls
in each of --rounds alternations, the blend forward's device time per view (srf_profile_*, render_fwd), and the peak
allocation over one call above the allocation before it.  The default points are the bench point (131 072 Gaussians,
512 x 512, 8 views), LaRa's Gaussian count (524 288) at 8 views and at the mesh extractor's 48 cameras.  Prints the card
name and power limit, then one JSON line per point.

    python tools/bench_forward_only.py [--iters 10] [--rounds 4] [--points 131072x8,524288x8,524288x48]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from timing import alternate, card, cuda_ms, peak_mib, summary  # noqa: E402  (tools/ is on sys.path as a script)


def run_point(P: int, V: int, H: int, W: int, iters: int, rounds: int) -> dict:
    from lara_b200 import _lib, rasterizer as R, scene as S
    dev = torch.device("cuda:0")
    sc = S.scene(P, 0)
    cams = S.cameras(V, H, W, 0)
    settings = [S.settings_for(c, torch.ones(3), sc["sh_degree"], dev, R.GaussianRasterizationSettings) for c in cams]
    camt = R.pack_cameras(settings, dev)
    t = {k: sc[k].to(dev).contiguous() for k in ("means3D", "shs", "opacities", "scales", "rotations")}

    def fwd(for_backward):
        return R.forward_views_raw(t["means3D"], t["shs"], None, t["opacities"], t["scales"], t["rotations"], None,
                                   camt, cams[0].tanfovx, cams[0].tanfovy, H, W, sc["sh_degree"],
                                   for_backward=for_backward)

    def settle():
        torch.cuda.synchronize()
        R._drain_ready(dev)

    # warm-up of both paths; the first call also sets the capacity high-water mark both paths then start from
    for fb in (True, False, True, False):
        fwd(fb)[3].resolve()
    settle()
    same = all(torch.equal(a, b) for a, b in zip(fwd(True)[:3], fwd(False)[:3]))
    settle()

    def timed(fn):
        # one call at a time, each to completion: an unresolved call keeps its state alive, so calls queued back to
        # back would hold several launch sets' workspaces at the 48-view point
        total = 0.0
        for _ in range(iters):
            total += cuda_ms(fn, 1)
            settle()
        return total / iters

    ms = alternate({True: lambda: fwd(True), False: lambda: fwd(False)}, rounds, timed)

    blend, peak, capacity = {}, {}, {}
    for fb in (True, False):
        _lib.profile_begin()
        fwd(fb)
        settle()
        blend[fb] = _lib.profile_end()["render_fwd"]
        out = []
        peak[fb] = round(peak_mib(lambda: out.append(fwd(fb))) * 2 ** 20)
        settle()
        capacity[fb] = out[0][3].capacity
        del out
        settle()
    name = {True: "training", False: "forward_only"}
    return {
        "point": {"P": P, "H": H, "W": W, "views": V, "capacity_per_view": capacity[False]},
        "outputs_bit_identical": same,
        "call_ms": {name[fb]: summary(ms[fb]) for fb in ms},
        "render_fwd_us_per_view": {name[fb]: 1000.0 * blend[fb][0] / V for fb in blend},
        "render_fwd_launches": {name[fb]: blend[fb][1] for fb in blend},
        "peak_bytes": {name[fb]: peak[fb] for fb in peak},
        "record_bytes": 8 * 4 * capacity[False] * V,
    }


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--points", default="131072x8,524288x8,524288x48", help="comma-separated PxV, 512 x 512 images")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_forward_only: needs a CUDA device")
    print(json.dumps({"card": card()}), flush=True)
    for p in args.points.split(","):
        P, V = (int(x) for x in p.split("x"))
        print(json.dumps(run_point(P, V, 512, 512, args.iters, args.rounds)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
