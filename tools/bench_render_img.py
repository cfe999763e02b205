"""Per-view cost of a full Renderer.render_img + loss backward (activations + rasterizer + epilogue):
   (a) the pipeline LaRa runs today: reference rasterizer (oracle/_ref) + torch epilogue,
   (b) drop-in: this repo's rasterizer under the unchanged torch epilogue,
   (c) lara_b200.renderer.Renderer: this rasterizer + fused epilogue, activations in torch,
   (d) the same with the activations fused into the preprocess kernels.

The four arms alternate within each of --repeats repeats of --iters views, timed with CUDA events.  Prints one line per
arm and one JSON line with the card's name and power limit.

    python tools/bench_render_img.py [P=524288] [--iters 30] [--repeats 5]
"""
import argparse
import json
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from timing import alternate, card, cuda_ms, summary  # noqa: E402  (tools/ is on sys.path as a script)


def loss_of(out):
    mask = (out["acc_map"] > 0).detach()
    return ((out["image"] - 0.4) ** 2).mean() + 1000.0 * out["rend_dist"].mean() + 0.1 * (out["depth"][..., 0] * mask).mean() \
        + 0.2 * (1 - (out["rend_normal"] * out["depth_normal"]).sum(-1)).mean()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("P", type=int, nargs="?", default=524288, help="Gaussians")
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    import diff_surfel_rasterization as DSR
    from lara_b200 import scene as S
    from lara_b200.renderer import Renderer
    from oracle import ref as REF
    from oracle.torch_restatements import render_img_epilogue_torch
    from test_epilogue import _inputs

    dev = torch.device("cuda:0")
    P, H, W = a.P, 512, 512
    ref = REF.load()
    sc = S.scene(P, 0)
    c = S.cameras(8, H, W, 0)[0]
    cam = types.SimpleNamespace(image_height=H, image_width=W, FoVx=0.75, FoVy=0.75,
                                world_view_transform=c.viewmatrix.to(dev), full_proj_transform=c.projmatrix.to(dev),
                                camera_center=c.campos.to(dev))
    _, _, rays, _ = _inputs(H, W, 3, dev)
    base = {"centers": sc["means3D"].to(dev), "shs": sc["shs"].to(dev),
            "opacity": torch.logit(sc["opacities"].clamp(1e-4, 1 - 1e-4)).to(dev),
            "scales": torch.log(sc["scales"]).to(dev), "rotations": (sc["rotations"] * 0.7).to(dev)}

    def torch_pipeline(mod):
        def run(raw):
            rs = S.settings_for(c, torch.ones(3), 1, dev, mod.GaussianRasterizationSettings)
            img, radii, allmap = mod.GaussianRasterizer(raster_settings=rs)(
                means3D=raw["centers"], means2D=torch.zeros_like(raw["centers"], requires_grad=True) + 0,
                shs=raw["shs"], opacities=torch.sigmoid(raw["opacity"]), scales=torch.exp(raw["scales"]),
                rotations=torch.nn.functional.normalize(raw["rotations"]), cov3D_precomp=None)
            return render_img_epilogue_torch(img, allmap, rays, cam.world_view_transform, 0.0)
        return run

    fast = Renderer(sh_degree=1, white_background=True)
    plain = Renderer(sh_degree=1, white_background=True, fused_activations=False)
    variants = {"reference rasterizer + torch epilogue (LaRa today)": torch_pipeline(ref),
                "lara_b200 rasterizer (drop-in) + torch epilogue": torch_pipeline(DSR),
                "lara_b200.renderer.Renderer, torch activations + fused epilogue":
                    lambda raw: plain.render_img(cam, rays, raw["centers"], raw["shs"], raw["opacity"], raw["scales"],
                                                 raw["rotations"], dev),
                "lara_b200.renderer.Renderer, fused activations + fused epilogue":
                    lambda raw: fast.render_img(cam, rays, raw["centers"], raw["shs"], raw["opacity"], raw["scales"],
                                                raw["rotations"], dev)}

    def step_of(fn):
        raw = {k: v.clone().requires_grad_(True) for k, v in base.items()}

        def step():
            for v in raw.values():
                v.grad = None
            loss_of(fn(raw)).backward()
        return step

    arms = {name: step_of(fn) for name, fn in variants.items()}
    for step in arms.values():
        for _ in range(5):
            step()
    times = alternate(arms, a.repeats, lambda step: cuda_ms(step, a.iters))
    res = {"card": card(), "P": P, "H": H, "W": W, "iters": a.iters}
    for name, ts in times.items():
        t = summary(ts)
        res[name] = {"view_ms": t}
        print(f"P={P} 512x512  {name:66s} {t['median']:7.3f} ms per view (render_img + loss.backward)")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
