"""Fused epilogue of LaRa's ``Renderer.render_img`` (SURVEY.md 8f rank 2) -- an additional entry
point next to the unchanged drop-in rasterizer.

``render_img_epilogue(color, allmap, rays, viewmatrix, depth_ratio, prex)`` returns exactly the
dict ``lightning/renderer_2dgs.py:256-268`` returns (same keys, shapes and -- permuted-view --
memory layout), computed by one CUDA kernel instead of ~12 torch ops, with a fused backward that
feeds ``dL_dcolor`` / ``dL_dallmap`` straight into the rasterizer's backward.  A maintainer can
switch ``Renderer.render_img`` to it with a two-line change::

    rendered_image, radii, allmap = rasterizer(...)            # unchanged
    if rays is None: return rendered_image.clamp(0, 1)
    return render_img_epilogue(rendered_image, allmap, rays, cam.world_view_transform, depth_ratio, prex)

One deliberate difference: where the reference's autograd produces NaN gradients (0/0 in the
backward of ``D / alpha`` at pixels with alpha == 0, 0 * inf where fp32 ``D / alpha`` overflows, 0 * NaN at a
non-finite median depth) the fused backward produces 0.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import _lib
from ._lib import _contig, _ptr


def epilogue_views_forward_raw(color, allmap, rays, cams, depth_ratio, image, depth, acc, rn, dn, dist):
    """The fused forward over V stacked views in one launch, enqueued on the current stream: color [V,3,H,W],
    allmap [V,8,H,W], rays [V,H,W,6] or None, cams [V,24] camera records (rasterizer.pack_cameras); outputs stacked
    [V,...] planar.  All tensors contiguous fp32 on one device.  Only the view matrix of each record is read, so for
    V = 1 a contiguous 16-float view matrix serves as `cams`."""
    V, H, W = int(color.shape[0]), int(color.shape[2]), int(color.shape[3])
    _lib.launch("srf_views_epilogue_forward", color.device, V, H, W, float(depth_ratio), color.data_ptr(),
                allmap.data_ptr(), _ptr(rays), cams.data_ptr(), image.data_ptr(), depth.data_ptr(), acc.data_ptr(),
                rn.data_ptr(), dn.data_ptr(), dist.data_ptr())


def epilogue_views_backward_raw(color, allmap, rays, cams, depth_ratio, gi, gd, ga, grn, gdn, gds):
    """Fused backward over V stacked views; returns (dL_dcolor [V,3,H,W], dL_dallmap [V,8,H,W])."""
    V, H, W = int(color.shape[0]), int(color.shape[2]), int(color.shape[3])
    dev = color.device
    scratch = torch.empty((V, 3, H, W), dtype=torch.float32, device=dev)
    d_color = torch.empty((V, 3, H, W), dtype=torch.float32, device=dev)
    d_allmap = torch.empty((V, 8, H, W), dtype=torch.float32, device=dev)
    _lib.launch("srf_views_epilogue_backward", dev, V, H, W, float(depth_ratio), color.data_ptr(), allmap.data_ptr(),
                _ptr(rays), cams.data_ptr(), _ptr(gi), _ptr(gd), _ptr(ga), _ptr(grn), _ptr(gdn), _ptr(gds),
                scratch.data_ptr(), d_color.data_ptr(), d_allmap.data_ptr())
    return d_color, d_allmap


def epilogue_forward_raw(color, allmap, rays, viewmatrix, depth_ratio, image, depth, acc, rn, dn, dist):
    """One view ([3,H,W], [8,H,W], rays [H,W,6] or None, a contiguous 16-float view matrix): the V = 1 case of
    :func:`epilogue_views_forward_raw`; outputs planar ([3,H,W], [1,H,W], [H,W], [3,H,W], [3,H,W], [H,W])."""
    epilogue_views_forward_raw(color[None], allmap[None], None if rays is None else rays[None], viewmatrix,
                               depth_ratio, image, depth, acc, rn, dn, dist)


def epilogue_backward_raw(color, allmap, rays, viewmatrix, depth_ratio, gi, gd, ga, grn, gdn, gds):
    """Backward of :func:`epilogue_forward_raw`; returns (dL_dcolor [3,H,W], dL_dallmap [8,H,W])."""
    d_color, d_allmap = epilogue_views_backward_raw(color[None], allmap[None], None if rays is None else rays[None],
                                                    viewmatrix, depth_ratio, gi, gd, ga, grn, gdn, gds)
    return d_color[0], d_allmap[0]


def _check_epilogue_inputs(color, allmap, rays, viewmatrix):
    """fp32 / CUDA / same-device / shape checks: the kernel takes raw pointers (the reference's torch ops
    would raise on their own)."""
    dev = color.device
    for name, t in (("rendered_image", color), ("allmap", allmap), ("world_view_transform", viewmatrix), ("rays", rays)):
        if t is None:
            continue
        if not t.is_cuda or t.device != dev:
            raise RuntimeError(f"render_img_epilogue: {name} must be a CUDA tensor on {dev}, got {t.device}")
        if t.dtype != torch.float32:
            raise RuntimeError(f"render_img_epilogue: expected scalar type Float but found {t.dtype} for {name}")
    H, W = int(color.shape[-2]), int(color.shape[-1])
    if color.ndim != 3 or color.shape[0] != 3 or tuple(allmap.shape) != (8, H, W):
        raise RuntimeError("render_img_epilogue: rendered_image must be [3,H,W] and allmap [8,H,W]")
    if rays is not None and tuple(rays.shape) != (H, W, 6):
        raise RuntimeError(f"render_img_epilogue: rays must be [H,W,6] = {(H, W, 6)}, got {tuple(rays.shape)}")
    if viewmatrix.numel() != 16:
        raise RuntimeError("render_img_epilogue: world_view_transform must have 16 elements")


class _Epilogue(torch.autograd.Function):
    @staticmethod
    def forward(ctx, color, allmap, rays, viewmatrix, depth_ratio):
        _check_epilogue_inputs(color, allmap, rays, viewmatrix)
        color = color.contiguous(); allmap = allmap.contiguous()
        viewmatrix = viewmatrix.contiguous()
        rays_c = rays.contiguous() if rays is not None else None
        H, W = int(color.shape[1]), int(color.shape[2])
        dev = color.device
        def new(*shape):
            return torch.empty(shape, dtype=torch.float32, device=dev)
        # separate planar tensors; the [H,W,C] permutes happen outside the Function so that the
        # results are ordinary autograd views (callers may then modify them in place)
        image, depth, acc, rn, dn, dist = new(3, H, W), new(1, H, W), new(H, W), new(3, H, W), new(3, H, W), new(H, W)
        epilogue_forward_raw(color, allmap, rays_c, viewmatrix, depth_ratio, image, depth, acc, rn, dn, dist)
        ctx.save_for_backward(color, allmap, rays_c if rays_c is not None else color.new_empty(0), viewmatrix)
        ctx.has_rays = rays_c is not None
        ctx.depth_ratio = float(depth_ratio)
        return image, depth, acc, rn, dn, dist

    @staticmethod
    def backward(ctx, g_image, g_depth, g_acc, g_rn, g_dn, g_dist):
        color, allmap, rays, viewmatrix = ctx.saved_tensors
        rays = rays if ctx.has_rays else None
        d_color, d_allmap = epilogue_backward_raw(color, allmap, rays, viewmatrix, ctx.depth_ratio, _contig(g_image),
                                                  _contig(g_depth), _contig(g_acc), _contig(g_rn), _contig(g_dn),
                                                  _contig(g_dist))
        return d_color, d_allmap, None, None, None


def render_img_epilogue(rendered_image: torch.Tensor, allmap: torch.Tensor, rays: Optional[torch.Tensor],
                        world_view_transform: torch.Tensor, depth_ratio: float = 0.0, prex: str = "") -> Dict[str, torch.Tensor]:
    """The dict of ``Renderer.render_img`` (renderer_2dgs.py:256-268) from the rasterizer's outputs."""
    image, depth, acc, rn, dn, dist = _Epilogue.apply(rendered_image, allmap, rays, world_view_transform, depth_ratio)
    return {
        f"image{prex}": image.permute(1, 2, 0), f"depth{prex}": depth.permute(1, 2, 0), f"acc_map{prex}": acc,
        f"rend_normal{prex}": rn.permute(1, 2, 0), f"depth_normal{prex}": dn.permute(1, 2, 0), f"rend_dist{prex}": dist,
    }
