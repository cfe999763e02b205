"""Batched multi-view entry (SURVEY.md 8f rank 1): all target views of one scene in one autograd node
AND one launch set.

LaRa's step renders the V target views of a scene one after the other (``lightning/network.py:486-495``:
``for j, c2w in enumerate(tar_c2ws): frame = self.gs_render.render_img(cam, rays_d, _centers, ...)``) and
then concatenates the frames (``:525``): V autograd nodes, V launch sets of ~8 kernels, V host round trips.
``render_scene_views`` is the same computation as one ``torch.autograd.Function`` over the ``srf_views_*``
entry points, whose kernels all carry a view dimension:

* forward : preprocess (grid.y = view) -> tile scan (one CTA per view) -> scatter -> per-tile sorts -> blend
            (one CTA per (tile, view), heaviest tiles first) -> fused epilogue (grid.z = view); outputs are
            stacked ``[V, C, H, W]`` buffers.  7 kernel launches + 1 memset per scene, no host wait.
* backward: fused epilogue backward (2 launches) -> blend backward over all (tile, view) -> per-Gaussian
            backward that sums the V views in registers and writes every parameter-gradient row once.

The per-view state (tile lists, records, ``n_contrib`` ...) is kept alive between the two phases, like the
reference keeps its three blobs in ``ctx`` (DSR ``__init__.py:97``).  An *additional* entry point: the
per-view drop-in API is unchanged.
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence

import torch

from . import _lib
from . import rasterizer as R
from .epilogue import epilogue_views_backward_raw, epilogue_views_forward_raw

OUT_KEYS = ("image", "depth", "acc_map", "rend_normal", "depth_normal", "rend_dist")


def shared_view_settings(settings_list: Sequence[R.GaussianRasterizationSettings]):
    """The settings every view of a batched call must share: (H, W, tanfovx, tanfovy, sh_degree, prefiltered, debug)."""
    s0 = settings_list[0]
    key = (int(s0.image_height), int(s0.image_width), float(s0.tanfovx), float(s0.tanfovy), int(s0.sh_degree))
    for rs in settings_list[1:]:
        if (int(rs.image_height), int(rs.image_width)) != key[:2]:
            raise RuntimeError("render_scene_views: all views of a call must share one image size")
        if (float(rs.tanfovx), float(rs.tanfovy)) != key[2:4] or int(rs.sh_degree) != key[4]:
            raise RuntimeError("render_scene_views: all views of a call must share the field of view and the SH degree")
    return key + (any(bool(rs.prefiltered) for rs in settings_list), any(bool(rs.debug) for rs in settings_list))


def _scene_views_forward(centers, shs, opacity, scales, rotations, rays, settings_list, depth_ratio, raw_activations,
                         for_backward):
    """Checks, the V-view rasterizer forward and the fused epilogue.  Returns the outputs (image, depth, acc, rn, dn,
    dist, radii) and what the backward needs: (inputs, rays, cams, color, allmap, state, geometry)."""
    dev = centers.device
    V = len(settings_list)
    centers_c, shs_c, _, opac_c, scales_c, rot_c, _ = R._normalise_inputs(
        centers, shs, None, opacity, scales, rotations, None)
    settings_list = [R._check_settings(rs, dev) for rs in settings_list]
    H, W, tfx, tfy, deg, prefiltered, debug = shared_view_settings(settings_list)
    rays_c = None
    if rays is not None:
        rays_c = rays.contiguous()
        if rays_c.dtype != torch.float32 or tuple(rays_c.shape) != (V, H, W, 6):
            raise RuntimeError(f"rays must be float32 [V,H,W,6] = {(V, H, W, 6)}, got {tuple(rays_c.shape)}")
        if rays_c.device != dev:
            raise RuntimeError(f"rays must live on {dev}, got {rays_c.device}")
    cams = R.pack_cameras(settings_list, dev)
    color, allmap, radii, state = R.forward_views_raw(
        centers_c, shs_c, None, opac_c, scales_c, rot_c, None, cams, tfx, tfy, H, W, deg,
        prefiltered=prefiltered, debug=debug, raw_activations=raw_activations, for_backward=for_backward)

    def new(*shape):
        return torch.empty(shape, dtype=torch.float32, device=dev)
    if rays_c is not None:
        image, depth, acc = new(V, 3, H, W), new(V, 1, H, W), new(V, H, W)
        rn, dn, dist = new(V, 3, H, W), new(V, 3, H, W), new(V, H, W)
        epilogue_views_forward_raw(color, allmap, rays_c, cams, depth_ratio, image, depth, acc, rn, dn, dist)
    else:
        image = color.clamp(0, 1)
        depth = acc = rn = dn = dist = centers_c.new_empty(0)
    return ((image, depth, acc, rn, dn, dist, radii),
            ((centers_c, shs_c, scales_c, rot_c), rays_c, cams, color, allmap, state, (H, W, tfx, tfy, deg, debug)))


class _RenderSceneViews(torch.autograd.Function):
    @staticmethod
    def forward(ctx, centers, shs, opacity, scales, rotations, rays, settings_list, depth_ratio, raw_activations):
        outs, (inputs, rays_c, cams, color, allmap, state, geometry) = _scene_views_forward(
            centers, shs, opacity, scales, rotations, rays, settings_list, depth_ratio, raw_activations, True)
        centers_c, shs_c, scales_c, rot_c = inputs
        radii = outs[-1]
        ctx.save_for_backward(centers_c, shs_c, scales_c, rot_c, rays_c if rays_c is not None else centers_c.new_empty(0),
                              cams, color, allmap, radii, state.geom, state.tile, state.image)
        ctx.state = state
        ctx.geometry = geometry
        ctx.has_rays = rays_c is not None
        ctx.depth_ratio = float(depth_ratio)
        ctx.raw_activations = bool(raw_activations)
        ctx.opac_shape = tuple(opacity.shape)
        ctx.mark_non_differentiable(radii)
        return outs

    @staticmethod
    def backward(ctx, g_image, g_depth, g_acc, g_rn, g_dn, g_dist, _g_radii):
        centers, shs, scales, rot, rays, cams, color, allmap, radii, _geom, _tile, _image = ctx.saved_tensors
        H, W, tfx, tfy, deg, debug = ctx.geometry

        if ctx.has_rays:
            c = _lib._contig
            d_color, d_allmap = epilogue_views_backward_raw(
                color, allmap, rays, cams, ctx.depth_ratio, c(g_image), c(g_depth), c(g_acc), c(g_rn), c(g_dn), c(g_dist))
        else:
            gi = g_image if g_image is not None else torch.zeros_like(color)
            d_color = (gi * ((color >= 0) & (color <= 1))).contiguous()      # vjp of clamp(0, 1)
            d_allmap = torch.zeros_like(allmap)
        g = R.backward_views_raw(ctx.state, radii, centers, shs, None, scales, rot, None, cams, tfx, tfy, H, W, deg,
                                 d_color, d_allmap, need_means2D=False, raw_activations=ctx.raw_activations, debug=debug)
        return (g["means3D"], g["sh"], g["opacities"].view(ctx.opac_shape), g["scales"], g["rotations"],
                None, None, None, None)


def render_scene_views(centers, shs, opacity, scales, rotations, settings_list: Sequence[R.GaussianRasterizationSettings],
                       rays: Optional[torch.Tensor] = None, depth_ratio: float = 0.0, raw_activations: bool = False,
                       streams: int = 1, prex: str = "") -> Dict[str, torch.Tensor]:
    """All views of one scene: returns stacked per-view results, ``{key+prex: [V, H, W, C] or [V, H, W]}`` with
    the keys, channel-last layout and values of ``Renderer.render_img``'s dict (renderer_2dgs.py:256-268) plus
    ``radii+prex`` [V, P]; ``out[k][j]`` is what the j-th ``render_img`` call of network.py:486-495 returns.
    ``rays=None``: only ``image`` as [V,3,H,W] (render_img's early return is the clamped planar image).
    ``streams`` is accepted for compatibility and ignored: the views share one launch set now.
    When no gradient can flow (``torch.no_grad()``, ``torch.inference_mode()``, no input requiring grad) the views
    take the forward-only path: the same values, without the backward's state and without an autograd node."""
    if len(settings_list) == 0:
        raise ValueError("render_scene_views needs at least one view")
    args = (centers, shs, opacity, scales, rotations, rays, list(settings_list), float(depth_ratio), bool(raw_activations))
    if R.needs_backward(centers, shs, opacity, scales, rotations, rays):
        image, depth, acc, rn, dn, dist, radii = _RenderSceneViews.apply(*args)
    else:
        (image, depth, acc, rn, dn, dist, radii), _ = _scene_views_forward(*args, False)
    if rays is None:          # render_img's early return hands back the clamped [3,H,W] image, not a dict
        return {f"image{prex}": image, f"radii{prex}": radii}
    return {
        f"image{prex}": image.permute(0, 2, 3, 1), f"depth{prex}": depth.permute(0, 2, 3, 1), f"acc_map{prex}": acc,
        f"rend_normal{prex}": rn.permute(0, 2, 3, 1), f"depth_normal{prex}": dn.permute(0, 2, 3, 1),
        f"rend_dist{prex}": dist, f"radii{prex}": radii,
    }


def concat_views(out: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """The layout LaRa's step hands to the loss: ``torch.cat([frame[k] for frame in views], dim=1)``
    (network.py:525), i.e. the views side by side along the width."""
    res = {}
    for k, t in out.items():
        if k.startswith("radii"):
            continue
        if t.ndim == 4:      # [V,H,W,C] -> [H, V*W, C]
            V, H, W, C = t.shape
            res[k] = t.permute(1, 0, 2, 3).reshape(H, V * W, C)
        else:                # [V,H,W] -> [H, V*W]
            V, H, W = t.shape
            res[k] = t.permute(1, 0, 2).reshape(H, V * W)
    return res
