"""One training step of LaRa's network on the fused path (DESIGN §3.28): ``Network`` + ``Losses``, forward and backward.

LaRa's base config (ViT-B/16, vol_embedding_reso 32, K = 2, 12 VolTransformer layers), B = 3 scenes of V = 8 target
views of 512^2, n_views 4, under bf16 autocast, seeded weights and a synthetic batch.  Two arms alternate in one run:

* ``records``: the camera records of all B*V views from ``batch_cameras``, one launch (``Network.forward`` as it is);
* ``minicam``: the coarse render's cameras built as LaRa builds them, one ``MiniCam`` per view through
  ``Renderer.render_batch_views`` (each with its device inverse, host projection matrix and copies).

Per step: the host-clock time around a device synchronise, kernel launches (a ``torch.profiler`` window of its own),
torch-visible synchronising calls (``torch.cuda.set_sync_debug_mode``), the peak-allocation increase, and the card's
name and power limit.  Prints one JSON line.

    python tools/bench_network.py [--repeats 7]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import types
import warnings

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from timing import alternate, card, host_ms, peak_mib, summary  # noqa: E402

B, V, H, W, N_VIEWS, ITER = 3, 8, 512, 512, 4, 5000


def base_cfg(n_views: int = N_VIEWS):
    """LaRa's configs/base.yaml model section."""
    model = types.SimpleNamespace(encoder_backbone="vit_base_patch16_224.dino", n_groups=[16], n_offset_groups=32, K=2,
                                  sh_degree=1, num_layers=12, num_heads=16, view_embed_dim=32, embedding_dim=256,
                                  vol_feat_reso=16, vol_embedding_reso=32, vol_embedding_out_dim=80)
    return types.SimpleNamespace(model=model, n_views=n_views, train=types.SimpleNamespace(use_rand_views=False))


def lara_batch(dev, B=B, V=V, H=H, W=W, seed=0, fov=0.6):
    """A collated LaRa batch on ``dev`` as ``assemble_batch`` leaves it: cameras on a sphere of radius ~2 looking at the
    origin, LaRa's intrinsics and rays, seeded images; ``fovx``, ``fovy``, ``near_far`` and ``meta`` on the device too,
    as after Lightning's transfer."""
    from lara_b200.batch import DOWN, fov_to_ixt, image_to_world
    from lara_b200.scene import look_at_c2w
    rng = np.random.default_rng(seed)
    c2w = np.stack([look_at_c2w(2 * np.pi * v / V + rng.uniform(0, 0.3), float(rng.uniform(-0.4, 0.4)),
                                float(rng.uniform(1.8, 2.2))).numpy() for _ in range(B) for v in range(V)])
    c2w = c2w.astype(np.float32).reshape(B, V, 4, 4)
    ixt = np.broadcast_to(fov_to_ixt(np.array([fov, fov], dtype=np.float32), np.array([H, W])), (B, V, 3, 3))

    def rays(scale, h, w):
        i2w = np.stack([image_to_world(c2w[b], ixt[b].copy(), scale) for b in range(B)])
        i2w = torch.from_numpy(i2w).to(dev, torch.float64)
        y, x = torch.meshgrid(torch.arange(h, device=dev), torch.arange(w, device=dev), indexing="ij")
        xyz = torch.stack([x + 0.5, y + 0.5, torch.ones_like(x, dtype=torch.float64)], -1).double()
        d = torch.einsum("hwj,bvji->bvhwi", xyz, i2w).float()
        o = torch.from_numpy(c2w[..., :3, 3]).to(dev)[:, :, None, None].expand(-1, -1, h, w, -1)
        return torch.cat([o, d], -1).contiguous()
    g = torch.Generator(device=dev).manual_seed(seed)
    c2w_t = torch.from_numpy(c2w).to(dev)
    return {"tar_rgb": torch.rand(B, V, H, W, 3, generator=g, device=dev), "tar_c2w": c2w_t,
            "tar_w2c": torch.inverse(c2w_t), "tar_ixt": torch.from_numpy(np.ascontiguousarray(ixt)).to(dev),
            "bg_color": torch.from_numpy(rng.choice([0.0, 0.5, 1.0], (B, V, 1)).repeat(3, -1).astype(np.float32)).to(dev),
            "tar_rays": rays(1.0, H, W), "tar_rays_down": rays(1.0 / DOWN, H // DOWN, W // DOWN),
            "near_far": torch.tensor([[1.2, 2.8]] * B, device=dev), "fovx": torch.full((B,), fov, device=dev),
            "fovy": torch.full((B,), fov, device=dev),
            "meta": {"tar_h": torch.full((B,), H, device=dev), "tar_w": torch.full((B,), W, device=dev)}}


class MiniCam:
    """LaRa's ``MiniCam`` (lightning/utils.py:22-48) step by step: ``torch.inverse`` of the pose on its device, the
    projection matrix filled on the host from the device field of view, both copied to the device."""

    def __init__(self, c2w, width, height, fovy, fovx, znear, zfar, device):
        self.image_width, self.image_height, self.FoVy, self.FoVx = width, height, fovy, fovx
        self.world_view_transform = torch.inverse(c2w).transpose(0, 1).to(device)
        proj = torch.zeros(4, 4)
        proj[0, 0], proj[1, 1] = 1 / torch.tan(fovx / 2), 1 / torch.tan(fovy / 2)
        proj[3, 2], proj[2, 2], proj[2, 3] = 1.0, zfar / (zfar - znear), -(zfar * znear) / (zfar - znear)
        self.projection_matrix = proj.transpose(0, 1).to(device)
        self.full_proj_transform = (self.world_view_transform @ self.projection_matrix).float()
        self.camera_center = -c2w[:3, 3].to(device)


def minicam_network(cfg):
    """``Network`` whose coarse render takes one ``MiniCam`` per view through ``Renderer.render_batch_views``, as LaRa's
    scene loop builds them (network.py:475-492)."""
    from lara_b200.network import Network

    class MiniCamNetwork(Network):
        def render_coarse(self, batch, cameras, gaussians):
            dev = batch["tar_c2w"].device
            cams = []
            for i in range(batch["tar_c2w"].shape[0]):
                znear, zfar = batch["near_far"][i]
                h, w = int(batch["meta"]["tar_h"][i]), int(batch["meta"]["tar_w"][i])
                cams.append([MiniCam(c2w, w, h, batch["fovy"][i], batch["fovx"][i], znear, zfar, dev)
                             for c2w in batch["tar_c2w"][i]])
            return self.gs_render.render_batch_views(cams, batch["tar_rays"], *gaussians, dev,
                                                     bg_colors=batch["bg_color"], keep_binning=True)
    return MiniCamNetwork(cfg)


def count_syncs(fn) -> int:
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum("synchronizing cuda operation" in str(x.message).lower() for x in w)


def launches(fn, steps=2) -> float:
    """Kernel launches per call of ``fn`` in a torch.profiler window of ``steps`` calls."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    n = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
            and "memcpy" not in e.name.lower() and "memset" not in e.name.lower())
    return n / steps


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    args = ap.parse_args()
    from lara_b200.loss import Losses
    from lara_b200.network import Network
    dev = torch.device("cuda:0")
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit']}", flush=True)
    torch.manual_seed(0)
    net = Network(base_cfg()).to(dev).train()
    torch.manual_seed(0)
    net_mc = minicam_network(base_cfg()).to(dev).train()
    net_mc.load_state_dict(net.state_dict())
    batch = lara_batch(dev)
    loss_fn = Losses()

    def step(model):
        model.zero_grad(set_to_none=True)
        torch.manual_seed(1)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = model(batch, with_fine=True)
            loss = loss_fn(batch, out, ITER)[0]
        loss.backward()
        return loss

    arms = {"records": lambda: step(net), "minicam": lambda: step(net_mc)}
    res = {"card": info, "B": B, "V": V, "H": H, "W": W, "n_views": N_VIEWS, "autocast": "bf16"}
    for fn in arms.values():          # warm-up of every shape the timed window uses
        fn()
    la, lb = float(arms["records"]()), float(arms["minicam"]())
    res["loss"] = {"records": la, "minicam": lb}
    samples = alternate(arms, args.repeats, host_ms)
    res["step_ms"] = {k: summary(v) for k, v in samples.items()}
    res["syncs_per_step"] = {k: count_syncs(fn) for k, fn in arms.items()}
    res["kernel_launches_per_step"] = {k: launches(fn) for k, fn in arms.items()}
    res["peak_mib"] = {k: peak_mib(fn) for k, fn in arms.items()}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
