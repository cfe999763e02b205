"""One LaRa scene-step of the renderer: V target views of one Gaussian set + loss + backward
(the loop of lightning/network.py:486-495, the cat of :525, a loss.py-like loss), ms per view:
   (a) LaRa today: reference rasterizer (oracle/_ref) + torch activations + torch epilogue, per view,
   (b) drop-in rasterizer under the same torch code, per view,
   (c) lara_b200.renderer.Renderer.render_img per view (fused activations + epilogue),
   (d) Renderer.render_views: one autograd node, one launch set for all views, torch loss on the concatenated layout,
   (e) Renderer.render_views + lara_b200.loss.scene_loss: the fused loss -> gradient-map producer on the stacked buffers."""
import os, sys, types
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from lara_b200 import scene as S
from oracle.torch_restatements import render_img_epilogue_torch
from lara_b200.multiview import concat_views
from lara_b200.loss import scene_loss
from lara_b200.renderer import Renderer
import diff_surfel_rasterization as DSR
from oracle import ref as REF
from test_epilogue import _inputs

dev = torch.device("cuda:0")
P = int(sys.argv[1]) if len(sys.argv) > 1 else 524288
V = int(sys.argv[2]) if len(sys.argv) > 2 else 8
H = W = 512
ref = REF.load()
sc = S.scene(P, 0)
cs = S.cameras(V, H, W, 0)
cams = [types.SimpleNamespace(image_height=H, image_width=W, FoVx=0.75, FoVy=0.75, world_view_transform=c.viewmatrix.to(dev),
                              full_proj_transform=c.projmatrix.to(dev), camera_center=c.campos.to(dev)) for c in cs]
rays = torch.stack([_inputs(H, W, 3 + v, dev)[2] for v in range(V)])
base = {"centers": sc["means3D"].to(dev), "shs": sc["shs"].to(dev), "opacity": torch.logit(sc["opacities"].clamp(1e-4, 1 - 1e-4)).to(dev),
        "scales": torch.log(sc["scales"]).to(dev), "rotations": (sc["rotations"] * 0.7).to(dev)}
tar = torch.rand((H, V * W, 3), device=dev)


def loss_of(out):
    return ((out["image"] - tar) ** 2).mean() + 1000.0 * out["rend_dist"].mean() \
        + 0.2 * ((1 - (out["rend_normal"] * out["depth_normal"]).sum(-1)) * out["acc_map"].detach()).mean()


def torch_loop(mod):
    def run(raw):
        frames = []
        for j, c in enumerate(cs):
            rs = S.settings_for(c, torch.ones(3), 1, dev, mod.GaussianRasterizationSettings)
            img, radii, allmap = mod.GaussianRasterizer(raster_settings=rs)(
                means3D=raw["centers"], means2D=torch.zeros_like(raw["centers"], requires_grad=True) + 0, shs=raw["shs"],
                opacities=torch.sigmoid(raw["opacity"]), scales=torch.exp(raw["scales"]),
                rotations=torch.nn.functional.normalize(raw["rotations"]), cov3D_precomp=None)
            frames.append(render_img_epilogue_torch(img, allmap, rays[j], cams[j].world_view_transform, 0.0))
        return {k: torch.cat([f[k] for f in frames], dim=1) for k in frames[0]}
    return run


fast = Renderer(sh_degree=1, white_background=True)


def fast_loop(raw):
    frames = [fast.render_img(cams[j], rays[j], raw["centers"], raw["shs"], raw["opacity"], raw["scales"], raw["rotations"], dev)
              for j in range(V)]
    return {k: torch.cat([f[k] for f in frames], dim=1) for k in frames[0]}


def batched(streams):
    return lambda raw: concat_views(fast.render_views(cams, rays, raw["centers"], raw["shs"], raw["opacity"], raw["scales"],
                                                      raw["rotations"], dev, streams=streams))


tar_views = tar.view(H, V, W, 3).permute(1, 0, 2, 3).contiguous()          # the batch's own [V,H,W,3] layout


def fused_loss_step(raw):
    out = fast.render_views(cams, rays, raw["centers"], raw["shs"], raw["opacity"], raw["scales"], raw["rotations"], dev)
    return scene_loss(out, tar_views, 5000)[0]


variants = [("LaRa today: reference rasterizer, torch activations + epilogue, per-view loop", torch_loop(ref)),
            ("drop-in rasterizer (lara_b200) under the same torch code", torch_loop(DSR)),
            ("Renderer.render_img per view (fused activations + epilogue)", fast_loop),
            ("Renderer.render_views (one launch set), torch loss on the concatenated layout", batched(1)),
            ("Renderer.render_views + fused scene_loss (no concat, one loss kernel each way)", None)]
for name, fn in variants:
    raw = {k: v.clone().requires_grad_(True) for k, v in base.items()}
    def step():
        for v in raw.values():
            v.grad = None
        (fused_loss_step(raw) if fn is None else loss_of(fn(raw))).backward()
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    N = 10
    for _ in range(N):
        step()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / N
    print(f"P={P} {V} views 512x512  {name:82s} {ms:8.3f} ms per scene-step  {ms / V:6.3f} ms per view")
