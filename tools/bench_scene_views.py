"""One LaRa scene-step of the renderer: V target views of one Gaussian set + loss + backward
(the loop of lightning/network.py:486-495, the cat of :525, a loss.py-like loss), ms per view:
   (a) LaRa today: reference rasterizer (oracle/_ref) + torch activations + torch epilogue, per view,
   (b) drop-in rasterizer under the same torch code, per view,
   (c) lara_b200.renderer.Renderer.render_img per view (fused activations + epilogue),
   (d) Renderer.render_views: one autograd node, one launch set for all views, torch loss on the concatenated layout,
   (e) Renderer.render_views + lara_b200.loss.scene_loss: the fused loss -> gradient-map producer on the stacked buffers.

The five arms alternate within each of --repeats repeats of --iters scene-steps, timed with CUDA events.  Prints one
line per arm and one JSON line with the card's name and power limit.

    python tools/bench_scene_views.py [P=524288] [V=8] [--iters 10] [--repeats 3]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("P", type=int, nargs="?", default=524288, help="Gaussians")
    ap.add_argument("V", type=int, nargs="?", default=8, help="target views")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    import diff_surfel_rasterization as DSR
    from lara_b200 import scene as S
    from lara_b200.loss import scene_loss
    from lara_b200.multiview import concat_views
    from lara_b200.renderer import Renderer
    from oracle import ref as REF
    from oracle.torch_restatements import render_img_epilogue_torch
    from test_epilogue import _inputs

    dev = torch.device("cuda:0")
    P, V, H, W = a.P, a.V, 512, 512
    ref = REF.load()
    sc = S.scene(P, 0)
    cs = S.cameras(V, H, W, 0)
    cams = [types.SimpleNamespace(image_height=H, image_width=W, FoVx=0.75, FoVy=0.75,
                                  world_view_transform=c.viewmatrix.to(dev), full_proj_transform=c.projmatrix.to(dev),
                                  camera_center=c.campos.to(dev)) for c in cs]
    rays = torch.stack([_inputs(H, W, 3 + v, dev)[2] for v in range(V)])
    base = {"centers": sc["means3D"].to(dev), "shs": sc["shs"].to(dev),
            "opacity": torch.logit(sc["opacities"].clamp(1e-4, 1 - 1e-4)).to(dev),
            "scales": torch.log(sc["scales"]).to(dev), "rotations": (sc["rotations"] * 0.7).to(dev)}
    tar = torch.rand((H, V * W, 3), device=dev)
    tar_views = tar.view(H, V, W, 3).permute(1, 0, 2, 3).contiguous()          # the batch's own [V,H,W,3] layout

    def loss_of(out):
        return ((out["image"] - tar) ** 2).mean() + 1000.0 * out["rend_dist"].mean() \
            + 0.2 * ((1 - (out["rend_normal"] * out["depth_normal"]).sum(-1)) * out["acc_map"].detach()).mean()

    def torch_loop(mod):
        def run(raw):
            frames = []
            for j, c in enumerate(cs):
                rs = S.settings_for(c, torch.ones(3), 1, dev, mod.GaussianRasterizationSettings)
                img, radii, allmap = mod.GaussianRasterizer(raster_settings=rs)(
                    means3D=raw["centers"], means2D=torch.zeros_like(raw["centers"], requires_grad=True) + 0,
                    shs=raw["shs"], opacities=torch.sigmoid(raw["opacity"]), scales=torch.exp(raw["scales"]),
                    rotations=torch.nn.functional.normalize(raw["rotations"]), cov3D_precomp=None)
                frames.append(render_img_epilogue_torch(img, allmap, rays[j], cams[j].world_view_transform, 0.0))
            return loss_of({k: torch.cat([f[k] for f in frames], dim=1) for k in frames[0]})
        return run

    fast = Renderer(sh_degree=1, white_background=True)

    def fast_loop(raw):
        frames = [fast.render_img(cams[j], rays[j], raw["centers"], raw["shs"], raw["opacity"], raw["scales"],
                                  raw["rotations"], dev) for j in range(V)]
        return loss_of({k: torch.cat([f[k] for f in frames], dim=1) for k in frames[0]})

    def batched(raw):
        return loss_of(concat_views(fast.render_views(cams, rays, raw["centers"], raw["shs"], raw["opacity"],
                                                      raw["scales"], raw["rotations"], dev, streams=1)))

    def fused_loss(raw):
        out = fast.render_views(cams, rays, raw["centers"], raw["shs"], raw["opacity"], raw["scales"], raw["rotations"],
                                dev)
        return scene_loss(out, tar_views, 5000)[0]

    variants = {"LaRa today: reference rasterizer, torch activations + epilogue, per-view loop": torch_loop(ref),
                "drop-in rasterizer (lara_b200) under the same torch code": torch_loop(DSR),
                "Renderer.render_img per view (fused activations + epilogue)": fast_loop,
                "Renderer.render_views (one launch set), torch loss on the concatenated layout": batched,
                "Renderer.render_views + fused scene_loss (no concat, one loss kernel each way)": fused_loss}

    def step_of(loss):
        raw = {k: v.clone().requires_grad_(True) for k, v in base.items()}

        def step():
            for v in raw.values():
                v.grad = None
            loss(raw).backward()
        return step

    arms = {name: step_of(loss) for name, loss in variants.items()}
    for step in arms.values():
        for _ in range(3):
            step()
    times = alternate(arms, a.repeats, lambda step: cuda_ms(step, a.iters))
    res = {"card": card(), "P": P, "views": V, "H": H, "W": W, "iters": a.iters}
    for name, ts in times.items():
        t = summary(ts)
        res[name] = {"scene_step_ms": t, "view_ms_median": t["median"] / V}
        print(f"P={P} {V} views 512x512  {name:82s} {t['median']:8.3f} ms per scene-step  "
              f"{t['median'] / V:6.3f} ms per view")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
