"""LaRa's ``Network`` (lightning/network.py:286-532) on the fused path: the whole B-scene forward with LaRa's
constructor, state dict and outputs, every stage one of this package's batched ops, and no scene loop (DESIGN §3.28).

* :class:`Network` -- ``Network(cfg, white_bkgd=True)``; ``state_dict()`` has exactly LaRa's keys, shapes and dtypes,
  so a checkpoint's ``net.*`` entries load strictly (:meth:`Network.from_lara_state_dict`).  Each LaRa tensor is one
  parameter here: the stage ops run on the modules the network owns (``dir_norm``, ``view_embed``, ``volume_grid``,
  ``decoder.*``), shared, never copied.
* :func:`concat_batch_views` -- LaRa's ``[B, H, V*W, C]`` layout of the outputs, for ``vis_images``.
"""
from __future__ import annotations

import math
import random
from typing import Dict, List

import numpy as np
import torch
from torch import nn

from .batch import batch_cameras
from .coarse_head import CoarseHead
from .feat_volume import FeatVolume, dense_grid
from .fine_head import FineHead
from .image_encoder import DinoEncoder
from .multiview import (OUT_KEYS, BatchCameras, FineSubset, render_batch_subset_views, render_batch_views)
from .point_feats import sample_batch_point_feats
from .renderer import Renderer
from .vol_transformer import VolTransformer

SCENE_SIZE = 0.5
OPACITY_SHIFT = -2.1792           # LaRa's opacity_shift (network.py:340)


class _Decoder(nn.Module):
    """LaRa's ``Decoder`` parameters under its names: ``mlp_coarse`` is the :class:`CoarseHead`'s module and ``norm``,
    ``cross_att``, ``mlp_fine`` the :class:`FineHead`'s, the same module objects."""

    def __init__(self, coarse: CoarseHead, fine: FineHead):
        super().__init__()
        self.mlp_coarse = coarse.mlp_coarse
        self.norm, self.cross_att, self.mlp_fine = fine.norm, fine.cross_att, fine.mlp_fine


def _scene_values(batch, B: int) -> List[List[float]]:
    """[fovx, fovy, tar_h, tar_w, render_img_scale] per scene as host floats: the device ones among them in one read."""
    scale = batch.get("render_img_scale", 1.0)
    cols = [batch["fovx"], batch["fovy"], batch["meta"]["tar_h"], batch["meta"]["tar_w"], scale]
    on_dev = [c for c in cols if isinstance(c, torch.Tensor) and c.is_cuda]
    read = iter(torch.cat([c.reshape(-1).double() for c in on_dev]).tolist()) if on_dev else None    # the host read
    out = []
    for c in cols:
        if isinstance(c, torch.Tensor) and c.is_cuda:
            vals = [next(read) for _ in range(c.numel())]
        else:
            vals = np.asarray(c.detach().cpu() if isinstance(c, torch.Tensor) else c, dtype=np.float64).reshape(-1)
            vals = vals.tolist()
        if len(vals) == 1:
            vals = vals * B
        if len(vals) != B:
            raise ValueError(f"Network.forward: one value per scene expected ({B}), got {len(vals)}")
        out.append(vals)
    return out


class Network(nn.Module):
    """LaRa's ``Network``: ``cfg`` is any object with LaRa's attribute paths (``cfg.model.*``, ``cfg.n_views``,
    ``cfg.train.use_rand_views``).  ``gs_render`` is :class:`lara_b200.renderer.Renderer`."""

    def __init__(self, cfg, white_bkgd: bool = True):
        super().__init__()
        m = cfg.model
        self.cfg = cfg
        self.scene_size = SCENE_SIZE
        self.white_bkgd = white_bkgd
        self.img_encoder = DinoEncoder(model_name=m.encoder_backbone, is_train=True)
        feat_dim = self.img_encoder.model.num_features
        self.grid_reso = m.vol_embedding_reso
        self.feat_vol_reso = m.vol_feat_reso
        feat_volume = FeatVolume(feat_dim, m.view_embed_dim, m.vol_feat_reso, scene_size=SCENE_SIZE)
        # registered in LaRa's order, so that state_dict() lists LaRa's keys in LaRa's order
        self.dir_norm = feat_volume.dir_norm
        self.register_buffer("dense_grid", dense_grid(self.grid_reso, SCENE_SIZE))
        self.register_buffer("centers", dense_grid(self.grid_reso * 2, SCENE_SIZE))
        if m.view_embed_dim > 0:
            self.view_embed = feat_volume.view_embed
        self.n_groups = m.n_groups
        self.vol_decoder = VolTransformer(
            embed_dim=m.embedding_dim, image_feat_dim=feat_dim + m.view_embed_dim, vol_low_res=self.grid_reso,
            vol_high_res=self.grid_reso * 2, out_dim=m.vol_embedding_out_dim, n_groups=self.n_groups,
            num_layers=m.num_layers, num_heads=m.num_heads)
        self.register_buffer("volume_grid", feat_volume.volume_grid)
        self.n_offset_groups = m.n_offset_groups
        self.register_buffer("group_centers", dense_grid(self.grid_reso * 2, SCENE_SIZE).reshape(1, -1, 3))

        self.sh_dim = (m.sh_degree + 1) ** 2 * 3
        self.scaling_dim, self.rotation_dim, self.opacity_dim = 2, 4, 1
        self.out_dim = self.sh_dim + self.scaling_dim + self.rotation_dim + self.opacity_dim
        self.K = m.K
        coarse = CoarseHead(m.vol_embedding_out_dim, self.sh_dim, self.K)
        fine = FineHead(m.vol_embedding_out_dim, self.sh_dim)
        self.decoder = _Decoder(coarse, fine)
        self.gs_render = Renderer(sh_degree=m.sh_degree, white_background=white_bkgd, radius=1)
        # the stage ops, not registered: their modules are the ones registered above
        self._stages = {"feat_volume": feat_volume, "coarse": coarse, "fine": fine}

        self.opacity_shift = OPACITY_SHIFT
        self.voxel_size = 2.0 / (self.grid_reso * 2)
        self.scaling_shift = np.log(0.5 * self.voxel_size / 3.0)

    @classmethod
    def from_lara_state_dict(cls, sd: Dict[str, torch.Tensor], cfg, white_bkgd: bool = True) -> "Network":
        """The network of a LaRa checkpoint's ``state_dict``: its ``net.*`` entries, loaded strictly."""
        net = cls(cfg, white_bkgd)
        net.load_state_dict({k[len("net."):]: v for k, v in sd.items() if k.startswith("net.")}, strict=True)
        return net

    def _feat_volume(self) -> FeatVolume:
        """The feature-volume op on this network's ``view_embed`` and ``volume_grid`` (``Module.to`` replaces
        buffers, and may replace parameters, so they are handed over at each call; ``dir_norm`` is shared)."""
        fv = self._stages["feat_volume"]
        fv.dir_norm = self.dir_norm
        fv.volume_grid = self.volume_grid
        if self.cfg.model.view_embed_dim > 0:
            fv.view_embed = self.view_embed
        return fv

    def n_views_sel(self) -> int:
        """The number of source views, drawn as LaRa draws it (network.py:434-437)."""
        if self.training:
            return random.randint(2, 4) if self.cfg.train.use_rand_views else self.cfg.n_views
        return self.cfg.n_views

    def render_geometry(self, batch, B: int):
        """(H, W, [(tan_fovx, tan_fovy)] per scene) of the render, from one host read: LaRa's ``int(tar_h *
        render_img_scale)`` and ``math.tan(fov * 0.5)`` (network.py:476-477, renderer_2dgs.set_rasterizer)."""
        fovx, fovy, th, tw, scale = _scene_values(batch, B)
        sizes = {(int(np.float32(h) * np.float32(s)), int(np.float32(w) * np.float32(s)))
                 for h, w, s in zip(th, tw, scale)}
        if len(sizes) != 1:
            raise ValueError(f"Network.forward: the scenes of a batch must share the render size, got {sorted(sizes)}")
        H, W = sizes.pop()
        return H, W, [(math.tan(fx * 0.5), math.tan(fy * 0.5)) for fx, fy in zip(fovx, fovy)]

    def render_coarse(self, batch, cameras: BatchCameras, gaussians):
        """The coarse render of all B*V target views, keeping the binning for the fine pass."""
        return render_batch_views(*gaussians, rays=batch["tar_rays"], raw_activations=self.gs_render.fused_activations,
                                  keep_binning=True, cameras=cameras)

    def forward(self, batch, with_fine: bool = False, return_buffer: bool = False) -> Dict[str, object]:
        """LaRa's ``Network.forward`` for all B scenes at once: ``{key: [B,V,H,W,C] or [B,V,H,W]}`` for LaRa's keys
        (``image``, ``depth``, ``acc_map``, ``rend_normal``, ``depth_normal``, ``rend_dist``, and with ``with_fine``
        the same with ``_fine``), plus ``render_pkg`` with ``return_buffer``: per scene the coarse tuple (centers, shs,
        opacity, scaling, rotation), then with ``with_fine`` the fine tuple (centers[mask], shs_fine, opacity, scaling,
        rotation, mask).  :func:`concat_batch_views` gives LaRa's ``[B,H,V*W,C]`` layout.

        Host reads: one, before any work is enqueued (the per-scene field of view and render size), plus
        ``FineSubset``'s one (two when a ``_check_mask`` branch fires) with ``with_fine``."""
        B, V, H_in, W_in, C = batch["tar_rgb"].shape
        H, W, tan_fov = self.render_geometry(batch, B)
        n_views_sel = self.n_views_sel()
        if V < n_views_sel:
            raise ValueError(f"Network.forward: the batch has {V} views, fewer than the {n_views_sel} source views")
        tar_rgb = batch["tar_rgb"]
        # a permuted view, fp32 also under autocast (where LaRa's einsum rounds the images to bf16)
        inps = tar_rgb[:, :n_views_sel].reshape(B * n_views_sel, H_in, W_in, C).permute(0, 3, 1, 2)
        img_feats = self.img_encoder.forward_maps(inps)

        fv = self._feat_volume()
        rays, w2cs, ixts = (batch[k][:, :n_views_sel] for k in ("tar_rays_down", "tar_w2c", "tar_ixt"))
        conds = [fv.cond_tokens(img_feats, rays, w2cs, ixts, (H_in, W_in), g) for g in self.n_groups]
        volume_feat_up = self.vol_decoder(conds)

        coarse, fine = self._stages["coarse"], self._stages["fine"]
        centers, shs, scaling, rotation, opacity = coarse.gaussians(
            volume_feat_up, self.group_centers, self.opacity_shift, self.scaling_shift,
            0.5 * self.scene_size / self.n_offset_groups)
        masks = (self.gs_render.opacity_activation(opacity).squeeze(-1) > 0.005).detach()

        cameras = BatchCameras(batch_cameras(batch["tar_c2w"], batch["bg_color"]), H, W, tan_fov,
                               self.gs_render.sh_degree)
        out_b = self.render_coarse(batch, cameras, (centers, shs, opacity, scaling, rotation))
        outputs = {k: out_b[k] for k in OUT_KEYS}
        if with_fine:
            sub = FineSubset(masks, check=True, training=self.training)
            img_ref = tar_rgb[:, :n_views_sel].permute(0, 1, 4, 2, 3)          # LaRa's _inps, read in place
            point_feats = sample_batch_point_feats(sub, centers, img_ref, out_b, w2cs, ixts)
            shs_fine = fine.fine_shs(volume_feat_up.view(B, -1, volume_feat_up.shape[-1]), self.K, sub, point_feats,
                                     shs)
            out_f = render_batch_subset_views(out_b["binning"], sub, shs_fine)
            outputs.update({k + "_fine": out_f[k + "_fine"] for k in OUT_KEYS})
        if return_buffer:
            pkg = []
            for b in range(B):
                pkg.append((centers[b], shs[b], opacity[b], scaling[b], rotation[b]))
                if with_fine:
                    lo, hi = sub.offsets[b], sub.offsets[b + 1]
                    pkg.append((centers[b].index_select(0, sub.idx[lo:hi]), shs_fine[lo:hi], opacity[b], scaling[b],
                                rotation[b], sub.masks[b]))
            outputs["render_pkg"] = pkg
        return outputs


def concat_batch_views(out: Dict[str, object]) -> Dict[str, torch.Tensor]:
    """LaRa's layout of :meth:`Network.forward`'s outputs, ``torch.cat`` of the views along the width
    (network.py:527-529): ``[B,V,H,W,C] -> [B,H,V*W,C]`` and ``[B,V,H,W] -> [B,H,V*W]``; other entries are left out."""
    res = {}
    for k, t in out.items():
        if k.startswith("radii") or not isinstance(t, torch.Tensor):
            continue
        if t.ndim == 5:
            B, V, H, W, C = t.shape
            res[k] = t.permute(0, 2, 1, 3, 4).reshape(B, H, V * W, C)
        elif t.ndim == 4:
            B, V, H, W = t.shape
            res[k] = t.permute(0, 2, 1, 3).reshape(B, H, V * W)
        else:
            raise ValueError(f"concat_batch_views: {k} must be [B,V,H,W,C] or [B,V,H,W], got {tuple(t.shape)}")
    return res


__all__ = ["Network", "concat_batch_views"]
