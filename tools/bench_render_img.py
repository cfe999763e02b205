"""Per-view cost of a full Renderer.render_img + loss backward (activations + rasterizer + epilogue):
   (a) the pipeline LaRa runs today: reference rasterizer (oracle/_ref) + torch epilogue,
   (b) drop-in: this repo's rasterizer under the unchanged torch epilogue,
   (c) lara_b200.renderer.Renderer: this rasterizer + fused epilogue, activations in torch,
   (d) the same with the activations fused into the preprocess kernels."""
import os, sys, time, types
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from lara_b200 import scene as S
from oracle.torch_restatements import render_img_epilogue_torch
from lara_b200.renderer import Renderer
import diff_surfel_rasterization as DSR
from oracle import ref as REF
from test_epilogue import _inputs

dev = torch.device("cuda:0")
P = int(sys.argv[1]) if len(sys.argv) > 1 else 524288
H = W = 512
ref = REF.load()
sc = S.scene(P, 0)
c = S.cameras(8, H, W, 0)[0]
cam = types.SimpleNamespace(image_height=H, image_width=W, FoVx=0.75, FoVy=0.75, world_view_transform=c.viewmatrix.to(dev),
                            full_proj_transform=c.projmatrix.to(dev), camera_center=c.campos.to(dev))
_, _, rays, _ = _inputs(H, W, 3, dev)
base = {"centers": sc["means3D"].to(dev), "shs": sc["shs"].to(dev), "opacity": torch.logit(sc["opacities"].clamp(1e-4, 1 - 1e-4)).to(dev),
        "scales": torch.log(sc["scales"]).to(dev), "rotations": (sc["rotations"] * 0.7).to(dev)}


def loss_of(out):
    mask = (out["acc_map"] > 0).detach()
    return ((out["image"] - 0.4) ** 2).mean() + 1000.0 * out["rend_dist"].mean() + 0.1 * (out["depth"][..., 0] * mask).mean() \
        + 0.2 * (1 - (out["rend_normal"] * out["depth_normal"]).sum(-1)).mean()


def torch_pipeline(mod):
    def run(raw):
        rs = S.settings_for(c, torch.ones(3), 1, dev, mod.GaussianRasterizationSettings)
        img, radii, allmap = mod.GaussianRasterizer(raster_settings=rs)(
            means3D=raw["centers"], means2D=torch.zeros_like(raw["centers"], requires_grad=True) + 0, shs=raw["shs"],
            opacities=torch.sigmoid(raw["opacity"]), scales=torch.exp(raw["scales"]),
            rotations=torch.nn.functional.normalize(raw["rotations"]), cov3D_precomp=None)
        return render_img_epilogue_torch(img, allmap, rays, cam.world_view_transform, 0.0)
    return run


fast = Renderer(sh_degree=1, white_background=True)
plain = Renderer(sh_degree=1, white_background=True, fused_activations=False)
variants = [("reference rasterizer + torch epilogue (LaRa today)", torch_pipeline(ref)),
            ("lara_b200 rasterizer (drop-in) + torch epilogue", torch_pipeline(DSR)),
            ("lara_b200.renderer.Renderer, torch activations + fused epilogue",
             lambda raw: plain.render_img(cam, rays, raw["centers"], raw["shs"], raw["opacity"], raw["scales"], raw["rotations"], dev)),
            ("lara_b200.renderer.Renderer, fused activations + fused epilogue",
             lambda raw: fast.render_img(cam, rays, raw["centers"], raw["shs"], raw["opacity"], raw["scales"], raw["rotations"], dev))]
for name, fn in variants:
    raw = {k: v.clone().requires_grad_(True) for k, v in base.items()}
    def step():
        for v in raw.values():
            v.grad = None
        loss_of(fn(raw)).backward()
    for _ in range(5):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    N = 30
    for _ in range(N):
        step()
    e1.record(); torch.cuda.synchronize()
    print(f"P={P} 512x512  {name:66s} {e0.elapsed_time(e1) / N:7.3f} ms per view (render_img + loss.backward)")
