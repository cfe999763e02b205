"""Plain-torch restatement of the coarse pass's feature-volume lifting in LaRa: ``Network.build_feat_vol``
(lightning/network.py:352-379, with ``projection`` :182-187, ``ray_to_plucker`` :414-423, ``ModLN`` :190-213 and
``rsh_cart_3``), the view-embedding concatenation of :451-452 and the block layout ``VolTransformer.forward`` builds
at :145-150.  The checker of lara_b200/csrc/feat_volume.cu.

The op sequence is LaRa's, so on the CPU in fp32 it reproduces LaRa's values and every gradient bit for bit
(tests/test_feat_volume.py).  The spherical-harmonic constants are written in closed form; in fp32 they round to the
same floats as LaRa's decimal literals.  In float64 the restatement stays in float64 (LaRa's ``.float()`` before
``grid_sample`` only lifts bf16 to fp32) and is the accuracy reference of the kernels.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

_PI = math.pi
_Y00 = 1.0 / (2.0 * math.sqrt(_PI))
_Y1 = math.sqrt(3.0 / (4.0 * _PI))
_Y2 = 0.5 * math.sqrt(15.0 / _PI)
_Y20A, _Y20B = 0.75 * math.sqrt(5.0 / _PI), 0.25 * math.sqrt(5.0 / _PI)
_Y22 = 0.25 * math.sqrt(15.0 / _PI)
_Y33 = 0.25 * math.sqrt(35.0 / (2.0 * _PI))
_Y32 = 0.5 * math.sqrt(105.0 / _PI)
_Y31 = math.sqrt(21.0 / (2.0 * _PI)) / 6.0                  # times (1.5 - 7.5 z^2)
_Y30A, _Y30B = 5.0 / 6.0 * math.sqrt(7.0 / _PI), math.sqrt(7.0 / _PI) / 3.0   # z (1.5 z^2 - 0.5) and z
_Y32B = 0.25 * math.sqrt(105.0 / _PI)


def rsh_cart_3(xyz):
    """Real spherical harmonics up to degree 3 of xyz [..., 3] -> [..., 16], index n (n+1) + m."""
    x, y, z = xyz[..., 0], xyz[..., 1], xyz[..., 2]
    x2, y2, z2 = x ** 2, y ** 2, z ** 2
    xy, xz, yz = x * y, x * z, y * z
    return torch.stack([
        xyz.new_tensor(_Y00).expand(xyz.shape[:-1]),
        -_Y1 * y, _Y1 * z, -_Y1 * x,
        _Y2 * xy, -_Y2 * yz, _Y20A * z2 - _Y20B, -_Y2 * xz, _Y22 * x2 - _Y22 * y2,
        -_Y33 * y * (3.0 * x2 - y2), _Y32 * xy * z, _Y31 * y * (1.5 - 7.5 * z2),
        _Y30A * z * (1.5 * z2 - 0.5) - _Y30B * z, _Y31 * x * (1.5 - 7.5 * z2), _Y32B * z * (x2 - y2),
        -_Y33 * x * (x2 - 3.0 * y2),
    ], -1)


def ray_to_plucker(rays):
    origin, direction = rays[..., :3], rays[..., 3:6]
    direction = F.normalize(direction, p=2.0, dim=-1)
    return torch.cat((direction, torch.cross(origin, direction, dim=-1)), dim=-1)


def mod_ln(x, cond, norm_w, norm_b, mlp_w, mlp_b):
    """ModLN.forward: LayerNorm(x; eps 1e-6) (1 + scale) + shift, (shift, scale) = Linear(SiLU(cond))."""
    shift, scale = F.linear(F.silu(cond), mlp_w, mlp_b).chunk(2, dim=-1)
    return F.layer_norm(x, (x.shape[-1],), norm_w, norm_b, 1e-6) * (1 + scale) + shift


def build_feat_vol_torch(img_feats, rays_down, w2cs, ixts, image_hw, volume_grid, params):
    """img_feats [B V,C,h,w], rays_down [B,V,h,w,6], w2cs [B,V,4,4], ixts [B,V,3,3], image_hw = (H_img, W_img),
    volume_grid [R,R,R,3], params = (norm.weight, norm.bias, mlp.1.weight, mlp.1.bias) -> [B,V,C,R,R,R]."""
    h, w = image_hw
    n_views_sel = rays_down.shape[1]
    src_ixts = ixts.reshape(-1, 3, 3)
    src_w2cs = w2cs.reshape(-1, 4, 4)
    img_wh = torch.tensor([w, h], device=img_feats.device)
    points = volume_grid.reshape(1, -1, 3) @ src_w2cs[:, :3, :3].permute(0, 2, 1) + src_w2cs[:, :3, 3][:, None]
    points = points @ src_ixts.permute(0, 2, 1)
    point_img = points[..., :2] / points[..., -1:]
    point_img = (point_img + 0.5) / img_wh * 2 - 1.0
    feats_dir = ray_to_plucker(rays_down).reshape(-1, *rays_down.shape[2:])
    feats_dir = torch.cat((rsh_cart_3(feats_dir[..., :3]), rsh_cart_3(feats_dir[..., 3:6])), dim=-1)
    x = torch.einsum("bchw->bhwc", img_feats)
    x = mod_ln(x, feats_dir, *params)
    x = torch.einsum("bhwc->bchw", x)
    n_channel = x.shape[1]
    lifted = x.to(torch.promote_types(x.dtype, torch.float32))
    feats_vol = F.grid_sample(lifted, point_img.unsqueeze(1).to(lifted.dtype), align_corners=False).to(x)
    R = volume_grid.shape[0]
    return feats_vol.view(-1, n_views_sel, n_channel, R, R, R)


def cond_tokens_torch(feat_vol, view_embed, n_group):
    """The view-embedding concatenation (network.py:451-452; view_embed [1,Vmax,E,1,1,1] or None) and the blocks
    VolTransformer.forward hands its layers (:145-150): [B,V,C,R,R,R] -> [B g^3, V bs^3, C+E]."""
    B, V, _, D, H, W = feat_vol.shape
    if view_embed is not None:
        feat_vol = torch.cat((feat_vol, view_embed[:, :V].expand(B, -1, -1, D, H, W)), dim=2)
    C = feat_vol.shape[2]
    bs = D // n_group
    blocks = feat_vol.unfold(3, bs, bs).unfold(4, bs, bs).unfold(5, bs, bs)
    blocks = blocks.contiguous().view(B, V, C, n_group ** 3, bs ** 3)
    return torch.einsum("bvcgl->bgvlc", blocks).reshape(B * n_group ** 3, bs ** 3 * V, C)
