"""Cost of the deterministic backward (DESIGN §3.13) at the bench point: 131 072 Gaussians, 512 x 512, 8 views.

One forward, then the default and the deterministic backward of it alternate in one process, each timed with CUDA
events over --iters calls.  Prints the card name and power limit, the per-call times, and the extra scratch of the
deterministic backward at LaRa's size (524 288 Gaussians, 8 views).

    python tools/bench_deterministic.py [--iters 20] [--rounds 4]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from timing import alternate, card, cuda_ms, summary  # noqa: E402  (tools/ is on sys.path when run as a script)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=4)
    args = ap.parse_args()
    from lara_b200 import _lib, rasterizer as R, scene as S
    lib = _lib.load()
    dev = torch.device("cuda:0")
    P, H, W, V = 131072, 512, 512, 8
    sc = S.scene(P, 0)
    cams = S.cameras(V, H, W, 0)
    settings = [S.settings_for(c, torch.ones(3), sc["sh_degree"], dev, R.GaussianRasterizationSettings) for c in cams]
    camt = R.pack_cameras(settings, dev)
    t = {k: sc[k].to(dev).contiguous() for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    ups = [S.upstream_grads(H, W, v, lara_like=True) for v in range(V)]
    gc = torch.stack([u[0] for u in ups]).to(dev).contiguous()
    ga = torch.stack([u[1] for u in ups]).to(dev).contiguous()
    color, allmap, radii, state = R.forward_views_raw(t["means3D"], t["shs"], None, t["opacities"], t["scales"],
                                                      t["rotations"], None, camt, cams[0].tanfovx, cams[0].tanfovy, H, W,
                                                      sc["sh_degree"])
    state.resolve()

    def bwd(det):
        R.backward_views_raw(state, radii, t["means3D"], t["shs"], None, t["scales"], t["rotations"], None, camt,
                             cams[0].tanfovx, cams[0].tanfovy, H, W, sc["sh_degree"], gc, ga, deterministic=det)

    arms = {"default": lambda: bwd(False), "deterministic": lambda: bwd(True)}
    for fn in (*arms.values(), *arms.values()):      # warm-up of both paths
        fn()
    res = {k: summary(v) for k, v in alternate(arms, args.rounds, lambda fn: cuda_ms(fn, args.iters)).items()}
    _lib.profile_begin()
    bwd(False)
    kd = _lib.profile_end()["render_bwd"]
    _lib.profile_begin()
    bwd(True)
    kt = _lib.profile_end()["render_bwd"]
    PL, VL = 524288, 8
    extra = _lib.det_backward_scratch_bytes(lib, VL, PL) - _lib.views_sizes(lib, VL, PL, 512, 512, 0)[5]
    out = {"card": card(), "point": {"P": P, "H": H, "W": W, "views": V},
           "backward_ms": res,
           "render_bwd_ms": {"default": kd[0], "default_launches": kd[1], "deterministic": kt[0],
                             "deterministic_launches": kt[1]},
           "ratio_median": res["deterministic"]["median"] / res["default"]["median"],
           "extra_scratch_bytes_lara": {"P": PL, "views": VL, "bytes": extra}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
