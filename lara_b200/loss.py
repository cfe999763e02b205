"""Fused loss -> dL/d(render_img outputs) producer (SURVEY.md 8f rank 3) -- an additional entry point.

LaRa's ``Losses.forward`` (``lightning/loss.py:33-60``) computes, on the ``[H, V*W, C]`` concatenation of a scene's
views, ``mean((image - tar_rgb)^2)`` (+ ``0.5 (1 - MS-SSIM)``) and, after iteration 1000,
``1000 mean(rend_dist) + 0.2 mean((1 - <rend_normal, depth_normal>) acc_map.detach())`` -- ~15 elementwise and
reduction kernels forward, ~20 in autograd, each a full-image HBM round trip, plus the ``torch.cat`` /
``permute`` copies that build the concatenated layout.  ``scene_loss`` computes the same terms directly on the
stacked planar ``[V,C,H,W]`` buffers that ``lara_b200.multiview.render_scene_views`` returns views of: one kernel
for the three sums, one kernel that writes the four gradient maps exactly where the fused epilogue's backward
reads them.  ``ms_ssim=True`` adds LaRa's ``0.5 (1 - MS-SSIM)`` term computed by the fused kernels of
``lara_b200.ssim`` on the planar views read as one ``H x V*W`` image (LaRa's layout); its gradient adds to ``g_image``
through autograd.
"""
from __future__ import annotations

from typing import Callable, Dict, Optional, Tuple

import torch

from . import _lib
from ._lib import _ptr
from .ssim import ms_ssim_views


def _planar(t: torch.Tensor) -> torch.Tensor:
    """[V,H,W,C] channel-last view of a planar buffer -> the planar [V,C,H,W] tensor (no copy for the views
    render_scene_views returns)."""
    return t.permute(0, 3, 1, 2).contiguous()


class _SceneLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, rend_normal, depth_normal, rend_dist, acc_map, target, with_reg, batch_scenes):
        dev = image.device
        V, _, H, W = image.shape
        for name, t in (("image", image), ("target", target), ("rend_normal", rend_normal), ("depth_normal", depth_normal),
                        ("rend_dist", rend_dist), ("acc_map", acc_map)):
            if t is None:
                continue
            if not t.is_cuda or t.device != dev or t.dtype != torch.float32 or not t.is_contiguous():
                raise RuntimeError(f"scene_loss: {name} must be a contiguous float32 CUDA tensor on {dev}")
        if tuple(target.shape) != (V, H, W, 3):
            raise RuntimeError(f"scene_loss: tar_rgb must be [V,H,W,3] = {(V, H, W, 3)}, got {tuple(target.shape)}")
        sums = torch.empty(3, dtype=torch.float64, device=dev)
        # partial sums reduced in a fixed order instead of atomics
        ws = (torch.empty(_lib.det_loss_workspace_bytes(_lib.load(), V, H, W) // 8, dtype=torch.float64, device=dev)
              if _lib.deterministic() else None)
        _lib.launch("srf_loss_forward", dev, V, H, W, 1 if with_reg else 0, image.data_ptr(), target.data_ptr(),
                    _ptr(rend_normal), _ptr(depth_normal), _ptr(acc_map), _ptr(rend_dist), sums.data_ptr(), _ptr(ws))
        npx = float(batch_scenes) * V * H * W
        mse = sums[0] / (3.0 * npx)
        dist = sums[1] / npx
        nerr = sums[2] / npx
        loss = mse + (1000.0 * dist + 0.2 * nerr if with_reg else 0.0)
        ctx.save_for_backward(image, target, rend_normal if with_reg else image.new_empty(0),
                              depth_normal if with_reg else image.new_empty(0), acc_map if with_reg else image.new_empty(0))
        ctx.with_reg, ctx.npx = bool(with_reg), npx
        return loss.float(), mse.float(), dist.float(), nerr.float()

    @staticmethod
    def backward(ctx, g_loss, _g_mse, _g_dist, _g_nerr):
        image, target, rn, dn, acc = ctx.saved_tensors
        dev = image.device
        V, _, H, W = image.shape
        up = g_loss.to(torch.float32).contiguous()
        g_image = torch.empty_like(image)
        if ctx.with_reg:
            g_rn, g_dn = torch.empty_like(rn), torch.empty_like(dn)
            g_dist = torch.empty((V, H, W), dtype=torch.float32, device=dev)
        else:
            g_rn = g_dn = g_dist = None
        _lib.launch("srf_loss_backward", dev, V, H, W, 1 if ctx.with_reg else 0, 1.0 / (3.0 * ctx.npx),
                    1000.0 / ctx.npx, 0.2 / ctx.npx, image.data_ptr(), target.data_ptr(),
                    _ptr(rn if ctx.with_reg else None), _ptr(dn if ctx.with_reg else None),
                    _ptr(acc if ctx.with_reg else None), up.data_ptr(), g_image.data_ptr(), _ptr(g_rn), _ptr(g_dn),
                    _ptr(g_dist))
        return g_image, g_rn, g_dn, g_dist, None, None, None, None


def scene_loss(out: Dict[str, torch.Tensor], tar_rgb: torch.Tensor, iter: int, batch_scenes: int = 1,
               ssim: Optional[Callable[[torch.Tensor, torch.Tensor], torch.Tensor]] = None,
               prex: str = "", ms_ssim: bool = False) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """One scene's contribution to ``Losses.forward`` (lightning/loss.py:17-62) from the stacked dict of
    ``render_scene_views`` / ``Renderer.render_views``: ``out[k]`` are ``[V,H,W,C]`` / ``[V,H,W]``, ``tar_rgb`` is the
    batch's ``[V,H,W,3]`` target (``batch['tar_rgb'][i]``).  ``batch_scenes`` = B of the batch (the reference's means run
    over all scenes).
    ``ms_ssim=True`` adds this scene's share of LaRa's MS-SSIM term, ``(0.5 / B) (1 - mean_c value_c)``, with the
    views side by side as one ``H x V*W`` image exactly as LaRa computes it (windows straddle the seams), and sets the
    stat ``ssim`` to ``mean_c value_c / B`` (summed over the scenes: LaRa's stat).
    ``ssim(image[V,3,H,W], target[V,3,H,W]) -> scalar`` adds ``0.5 (1 - ssim)``; it receives the per-view stack, which
    is not LaRa's layout, so the library's MS-SSIM plugged in here gives a different number from LaRa's.
    Returns (loss, scalar_stats) with the reference's stat names."""
    if ms_ssim and ssim is not None:
        raise ValueError("scene_loss: pass either ms_ssim=True or ssim=, not both")
    with_reg = f"rend_dist{prex}" in out and iter > 1000 and prex != "_fine"
    image = _planar(out[f"image{prex}"])
    rn = _planar(out[f"rend_normal{prex}"]) if with_reg else None
    dn = _planar(out[f"depth_normal{prex}"]) if with_reg else None
    dist = out[f"rend_dist{prex}"].contiguous() if with_reg else None
    acc = out[f"acc_map{prex}"].detach().contiguous() if with_reg else None
    loss, mse, distortion, nerr = _SceneLoss.apply(image, rn, dn, dist, acc, tar_rgb.contiguous(), with_reg, int(batch_scenes))
    stats = {f"mse{prex}": mse.detach(), f"psnr{prex}": -10.0 * torch.log10(mse.detach())}
    if ssim is not None:
        s = ssim(image, tar_rgb.permute(0, 3, 1, 2))
        stats[f"ssim{prex}"] = s.detach()
        loss = loss + 0.5 * (1 - s)
    if ms_ssim:
        s = ms_ssim_views(image, tar_rgb.permute(0, 3, 1, 2))
        stats[f"ssim{prex}"] = s.detach() / batch_scenes
        loss = loss + (0.5 / batch_scenes) * (1 - s)
    if with_reg:
        stats[f"distortion{prex}"] = distortion.detach()
        stats[f"normal{prex}"] = nerr.detach()
    return loss, stats
