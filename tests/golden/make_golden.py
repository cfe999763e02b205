"""Generate the golden fixtures in tests/golden/*.npz by running the UNMODIFIED reference
rasterizer (oracle/_ref, built by oracle/build_ref.py).  The committed files were made with the reference's
sm_100 build on a B200; this package reproduces them bit for bit (its fp32 operation order is that build's).

    python tests/golden/make_golden.py OUT_DIR
    cp OUT_DIR/*.npz tests/golden/

The reference ships no fixtures for this path (SURVEY.md 8c), so these files are what
pins the CPU oracle (tests/test_oracle_golden.py) and, on the GPU, the product.  Each
file holds the case name, the camera, the reference's outputs, its internal state (radii, tiles_touched,
sorted point list, tile ranges, n_contrib) and its gradients for fixed upstream grads; the scene and the upstream
grads are regenerated from their seeds (tests/helpers.load_golden).
Gradients use fp32 atomics in the reference and therefore carry run-to-run noise at the
1e-6 relative level; `grad_noise` records the measured ref-vs-ref difference.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from lara_b200 import scene as S  # noqa: E402
from oracle import ref as REF  # noqa: E402


def case_inputs(name: str):
    """Deterministic small scenes covering the reference's branches."""
    if name == "basic_sh1":
        sc = S.scene(2048, 0, sh_degree=1)
        cam = S.cameras(3, 64, 64, 0)[0]
        bg = [1.0, 1.0, 1.0]
    elif name == "ragged_sh3":
        sc = S.scene(3000, 1, sh_degree=3)
        cam = S.cameras(3, 50, 72, 1)[1]      # H=50, W=72: not multiples of 16
        bg = [0.5, 0.5, 0.5]
    elif name == "culled_ties_sh0":
        sc = S.scene(1024, 2, sh_degree=0)
        cam = S.cameras(3, 64, 64, 2)[2]
        # exact duplicates -> identical depth bits in the same tiles: exercises sort stability
        for k in ("means3D", "scales", "rotations", "opacities", "shs"):
            sc[k][64:128] = sc[k][0:64]
        # a slab of Gaussians behind / too close to the camera -> frustum culled
        sc["means3D"][900:1024] = sc["means3D"][900:1024] * 0.1 + cam.c2w[:3, 3] * 1.02
        # a few large, opaque splats -> early termination and >256 instances in a tile
        sc["scales"][0:8] = 0.25
        sc["opacities"][0:8] = 0.99
        sc["opacities"][8:16] = 1e-4           # never reaches alpha 1/255
        bg = [0.0, 0.0, 0.0]
    else:
        raise KeyError(name)
    return sc, cam, torch.tensor(bg, dtype=torch.float32)


CASES = ["basic_sh1", "ragged_sh3", "culled_ties_sh0"]


def upstream_grads_for(cam):
    return S.upstream_grads(cam.image_height, cam.image_width, 7)


def main(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    ref = REF.load()
    dev = torch.device("cuda:0")
    for name in CASES:
        sc, cam, bg = case_inputs(name)
        H, W = cam.image_height, cam.image_width
        scd = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in sc.items()}
        st = S.settings_for(cam, bg, sc["sh_degree"], dev, ref.GaussianRasterizationSettings)
        r = REF.forward_raw(ref, scd, st)
        gc, ga = upstream_grads_for(cam)

        def grads():
            leaves = {k: scd[k].clone().requires_grad_(True) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
            m2d = torch.zeros_like(leaves["means3D"], requires_grad=True)
            rast = ref.GaussianRasterizer(raster_settings=st)
            c, rd, am = rast(means3D=leaves["means3D"], means2D=m2d, shs=leaves["shs"], opacities=leaves["opacities"],
                             scales=leaves["scales"], rotations=leaves["rotations"])
            torch.autograd.backward((c, am), (gc.to(dev), ga.to(dev)))
            g = {k: v.grad.cpu().numpy() for k, v in leaves.items()}
            g["means2D"] = m2d.grad.cpu().numpy()
            return g

        g1, g2 = grads(), grads()
        noise = {k: float(np.abs(g1[k] - g2[k]).max() / max(np.abs(g1[k]).max(), 1e-30)) for k in g1}
        vis = (r["radii"] > 0).cpu().numpy()
        np.savez_compressed(
            os.path.join(out_dir, name + ".npz"),
            # inputs (the scene and the upstream grads follow from `case`)
            case=np.str_(name), sh_degree=np.int32(sc["sh_degree"]),
            viewmatrix=cam.viewmatrix.numpy(), projmatrix=cam.projmatrix.numpy(), campos=cam.campos.numpy(),
            tanfovx=np.float64(cam.tanfovx), tanfovy=np.float64(cam.tanfovy), H=np.int32(H), W=np.int32(W),
            bg=bg.numpy(),
            # reference outputs and state
            color=r["color"].cpu().numpy(), allmap=r["allmap"].cpu().numpy(), radii=r["radii"].cpu().numpy(),
            num_rendered=np.int64(r["num_rendered"]), tiles_touched=r["tiles_touched"].cpu().numpy(),
            point_list=r["point_list"].cpu().numpy(), ranges=r["ranges"].cpu().numpy(),
            n_contrib=r["n_contrib"].cpu().numpy(), accum=r["accum"].cpu().numpy(),
            depths=np.where(vis, r["depths"].cpu().numpy(), 0).astype(np.float32),
            transMat=np.where(vis[:, None], r["transMat"].cpu().numpy(), 0).astype(np.float32),
            means2D=np.where(vis[:, None], r["means2D"].cpu().numpy(), 0).astype(np.float32),
            rgb=np.where(vis[:, None], r["rgb"].cpu().numpy(), 0).astype(np.float32),
            # reference gradients
            **{"g_" + k: v for k, v in g1.items()},
            grad_noise=np.array([noise[k] for k in sorted(noise)], dtype=np.float64),
        )
        print(name, "P", sc["means3D"].shape[0], "R", r["num_rendered"], "visible", int(vis.sum()), "noise", noise, flush=True)


if __name__ == "__main__":
    main(sys.argv[1])
