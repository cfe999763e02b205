"""Batched multi-view entry (SURVEY.md 8f rank 1): all target views of one scene in one autograd node
AND one launch set.

LaRa's step renders the V target views of a scene one after the other (``lightning/network.py:486-495``:
``for j, c2w in enumerate(tar_c2ws): frame = self.gs_render.render_img(cam, rays_d, _centers, ...)``) and
then concatenates the frames (``:525``): V autograd nodes, V launch sets of ~8 kernels, V host round trips.
``render_scene_views`` is the same computation as one ``torch.autograd.Function`` over the ``srf_scenes_*``
entry points (one scene), whose kernels all carry a view dimension:

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

from typing import Dict, NamedTuple, Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import _DeviceGuard, _ptr
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


def _epilogue_forward(color, allmap, rays_c, cams, depth_ratio):
    """The six render_img outputs of the rasterizer's stacked color / allmap (only the clamped image without rays)."""
    V, _, H, W = color.shape

    def new(*shape):
        return torch.empty(shape, dtype=torch.float32, device=color.device)
    if rays_c is not None:
        image, depth, acc = new(V, 3, H, W), new(V, 1, H, W), new(V, H, W)
        rn, dn, dist = new(V, 3, H, W), new(V, 3, H, W), new(V, H, W)
        epilogue_views_forward_raw(color, allmap, rays_c, cams, depth_ratio, image, depth, acc, rn, dn, dist)
    else:
        image = color.clamp(0, 1)
        depth = acc = rn = dn = dist = color.new_empty(0)
    return image, depth, acc, rn, dn, dist


def _epilogue_backward(color, allmap, rays, cams, depth_ratio, has_rays, g_image, g_depth, g_acc, g_rn, g_dn, g_dist):
    """dL/dcolor and dL/dallmap from the gradients of the six outputs of :func:`_epilogue_forward`."""
    if has_rays:
        c = _lib._contig
        return epilogue_views_backward_raw(color, allmap, rays, cams, depth_ratio, c(g_image), c(g_depth), c(g_acc),
                                           c(g_rn), c(g_dn), c(g_dist))
    gi = g_image if g_image is not None else torch.zeros_like(color)
    d_color = (gi * ((color >= 0) & (color <= 1))).contiguous()      # vjp of clamp(0, 1)
    return d_color, torch.zeros_like(allmap)


def _views_forward(inputs, rays_c, cams, geometry, prefiltered, depth_ratio, raw_activations, for_backward,
                   keep_list=False):
    """The rasterizer forward of the S*V views of S scenes and the fused epilogue: ``inputs`` the checked [S,P,...]
    centers, shs, opacity, scales and rotations, ``cams`` the [S*V, SRF_CAM_FLOATS] camera records (scene s's views are
    s*V .. s*V+V-1), ``geometry`` (H, W, tan_fovx per scene, tan_fovy per scene, sh degree, debug), ``rays_c``
    [S*V,H,W,6] or None.  Returns the outputs (image, depth, acc, rn, dn, dist, radii) stacked [S*V, ...] and (cams,
    color, allmap, state)."""
    H, W, tfx, tfy, deg, debug = geometry
    dev = inputs[0].device
    centers, shs, opacity, scales, rotations = inputs
    with _DeviceGuard(dev):
        color, allmap, radii, state = R.forward_batch_raw(
            centers, shs, None, opacity, scales, rotations, None, cams, list(zip(tfx, tfy)), H, W, deg,
            prefiltered=prefiltered, debug=debug, raw_activations=raw_activations, for_backward=for_backward, keep_list=keep_list)
        outs = (*_epilogue_forward(color, allmap, rays_c, cams, depth_ratio), radii)
    return outs, (cams, color, allmap, state)


class _RenderSceneViews(torch.autograd.Function):
    """One autograd node over the S*V views of S scenes (arguments as :func:`_views_forward`); the gradients of the
    [S,P,...] inputs are each scene's sum over its own views."""

    @staticmethod
    def forward(ctx, centers, shs, opacity, scales, rotations, rays_c, cams, geometry, prefiltered, depth_ratio,
                raw_activations, keep=None):
        outs, (cams, color, allmap, state) = _views_forward(
            (centers, shs, opacity, scales, rotations), rays_c, cams, geometry, prefiltered, depth_ratio,
            raw_activations, True)
        if keep is not None:
            keep.append((cams, state))
        radii = outs[-1]
        ctx.save_for_backward(centers, shs, scales, rotations, rays_c if rays_c is not None else color.new_empty(0),
                              cams, color, allmap, radii, state.geom, state.tile, state.image)
        ctx.state, ctx.geometry, ctx.has_rays = state, geometry, rays_c is not None
        ctx.depth_ratio, ctx.raw_activations, ctx.opac_shape = float(depth_ratio), bool(raw_activations), tuple(opacity.shape)
        ctx.mark_non_differentiable(radii)
        return outs

    @staticmethod
    def backward(ctx, g_image, g_depth, g_acc, g_rn, g_dn, g_dist, _g_radii):
        centers, shs, scales, rot, rays, cams, color, allmap, radii, _geom, _tile, _image = ctx.saved_tensors
        H, W, tfx, tfy, deg, debug = ctx.geometry
        d_color, d_allmap = _epilogue_backward(color, allmap, rays, cams, ctx.depth_ratio, ctx.has_rays, g_image, g_depth,
                                               g_acc, g_rn, g_dn, g_dist)
        g = R.backward_batch_raw(ctx.state, radii, centers, shs, scales, rot, cams, list(zip(tfx, tfy)), H, W, deg,
                                 d_color, d_allmap,
                                 raw_activations=ctx.raw_activations, debug=debug)
        return (g["means3D"], g["sh"], g["opacities"].view(ctx.opac_shape), g["scales"], g["rotations"],
                None, None, None, None, None, None, None)


def _render_views(inputs, rays_c, cams, geometry, prefiltered, depth_ratio, raw_activations, keep_binning, tensors):
    """:class:`_RenderSceneViews` when a gradient can flow, else the forward-only path; returns the outputs of
    :func:`_views_forward` and, with ``keep_binning``, the :class:`SceneBinning` of the call (``tensors``: the caller's
    five Gaussian tensors), else None."""
    keep = [] if keep_binning else None
    if R.needs_backward(*tensors, rays_c):
        outs = _RenderSceneViews.apply(*inputs, rays_c, cams, geometry, prefiltered, depth_ratio, raw_activations,
                                       keep)
    else:
        outs, (cams, _, _, state) = _views_forward(inputs, rays_c, cams, geometry, prefiltered, depth_ratio,
                                                   raw_activations, False, keep_list=keep_binning)
        if keep is not None:
            keep.append((cams, state))
    if not keep_binning:
        return outs, None
    cams, state = keep[0]
    return outs, SceneBinning(state, outs[-1], inputs[0], cams, geometry, rays_c, depth_ratio, raw_activations, tensors)


def render_scene_views(centers, shs, opacity, scales, rotations, settings_list: Sequence[R.GaussianRasterizationSettings],
                       rays: Optional[torch.Tensor] = None, depth_ratio: float = 0.0, raw_activations: bool = False,
                       streams: int = 1, prex: str = "", keep_binning: bool = False) -> Dict[str, object]:
    """All views of one scene: returns stacked per-view results, ``{key+prex: [V, H, W, C] or [V, H, W]}`` with
    the keys, channel-last layout and values of ``Renderer.render_img``'s dict (renderer_2dgs.py:256-268) plus
    ``radii+prex`` [V, P]; ``out[k][j]`` is what the j-th ``render_img`` call of network.py:486-495 returns.
    ``rays=None``: only ``image`` as [V,3,H,W] (render_img's early return is the clamped planar image).
    ``streams`` is accepted for compatibility and ignored: the views share one launch set now.
    When no gradient can flow (``torch.no_grad()``, ``torch.inference_mode()``, no input requiring grad) the views
    take the forward-only path: the same values, without the backward's state and without an autograd node.
    ``keep_binning=True`` adds ``out["binning"+prex]``, an opaque :class:`SceneBinning` that
    :func:`render_subset_views` renders a masked subset of these Gaussians from."""
    if len(settings_list) == 0:
        raise ValueError("render_scene_views needs at least one view")
    dev = centers.device
    V = len(settings_list)
    centers_c, shs_c, _, opac_c, scales_c, rot_c, _ = R._normalise_inputs(
        centers, shs, None, opacity, scales, rotations, None)
    settings = [R._check_settings(rs, dev) for rs in settings_list]
    H, W, tfx, tfy, deg, prefiltered, debug = shared_view_settings(settings)
    rays_c = None
    if rays is not None:
        rays_c = rays.contiguous()
        if rays_c.dtype != torch.float32 or tuple(rays_c.shape) != (V, H, W, 6):
            raise RuntimeError(f"rays must be float32 [V,H,W,6] = {(V, H, W, 6)}, got {tuple(rays_c.shape)}")
        if rays_c.device != dev:
            raise RuntimeError(f"rays must live on {dev}, got {rays_c.device}")
    # one scene: S = 1, whose [S*V, ...] outputs are the [V, ...] ones.  With P = 0 the checks read the empty scales and
    # rotations as absent; the node takes the caller's empty tensors instead, which then receive empty gradients
    inputs = tuple(None if t is None else t.unsqueeze(0)
                   for t in (centers_c, shs_c, opac_c, scales if scales_c is None else scales_c,
                             rotations if rot_c is None else rot_c))
    outs, binning = _render_views(inputs, rays_c, _pack(settings, dev), (H, W, (tfx,), (tfy,), deg, debug), prefiltered,
                                  float(depth_ratio), bool(raw_activations), keep_binning,
                                  (centers, shs, opacity, scales, rotations))
    out = _out_dict(*outs, rays is not None, prex)
    if binning is not None:
        out["binning" + prex] = binning
    return out


def _pack(settings, dev):
    """The camera records of checked view settings (``rasterizer.pack_cameras``), built outside autograd."""
    with torch.no_grad():
        return R.pack_cameras(settings, dev)


def _out_dict(image, depth, acc, rn, dn, dist, radii, has_rays, prex):
    if not has_rays:          # render_img's early return hands back the clamped [3,H,W] image, not a dict
        return {f"image{prex}": image, f"radii{prex}": radii}
    return {
        f"image{prex}": image.permute(0, 2, 3, 1), f"depth{prex}": depth.permute(0, 2, 3, 1), f"acc_map{prex}": acc,
        f"rend_normal{prex}": rn.permute(0, 2, 3, 1), f"depth_normal{prex}": dn.permute(0, 2, 3, 1),
        f"rend_dist{prex}": dist, f"radii{prex}": radii,
    }


class SceneBinning:
    """What a ``render_scene_views`` / ``render_batch_views(..., keep_binning=True)`` call leaves for
    :func:`render_subset_views` / :func:`render_batch_subset_views`: the coarse forward's state (records, depths, tile
    rectangles, radii and depth-sorted tile lists of every view), its ``scenes`` S, the checked centers ([P,3] or
    [S,P,3]), its cameras, geometry (H, W, tan_fovx and tan_fovy per scene, SH degree, debug), rays, ``depth_ratio`` and
    ``raw_activations`` flag, and the caller's five Gaussian tensors with their ``_version`` at the call.  Opaque: hand
    it to the subset render as it is."""
    __slots__ = ("state", "radii", "means", "scenes", "cams", "geometry", "rays", "depth_ratio", "raw_activations",
                 "tensors", "versions")

    def __init__(self, state, radii, means, cams, geometry, rays, depth_ratio, raw_activations, tensors):
        self.state, self.radii, self.means, self.cams, self.geometry = state, radii, means, cams, geometry
        self.scenes = int(means.shape[0]) if means.ndim == 3 else 1
        self.rays, self.depth_ratio, self.raw_activations, self.tensors = rays, depth_ratio, raw_activations, tensors
        # inference tensors keep no version counter (None: not checked)
        self.versions = tuple(None if t.is_inference() else t._version for t in tensors + (radii,))

    def check_unchanged(self):
        for name, t, v in zip(("centers", "shs", "opacity", "scales", "rotations", "radii"), self.tensors + (self.radii,),
                              self.versions):
            if v is not None and t._version != v:
                raise RuntimeError(f"render_subset_views: the coarse {name} was modified in place after the coarse "
                                   "render_scene_views call, so its binning no longer describes these Gaussians")


def _subset_forward(b: SceneBinning, idx, shs_c, for_backward, offsets=None, counts=None):
    """srf_scenes_subset_forward on the coarse state and the fused epilogue: ``idx`` the concatenated per-scene subsets,
    ``offsets`` / ``counts`` their device [S+1] bounds and host counts (None: one scene, its n = idx.numel()).  Returns
    the outputs (image, depth, acc, rn, dn, dist, radii [S*V, n_max]) and (color, allmap, state) for the backward."""
    lib = _lib.load()
    st = b.state
    dev = b.means.device
    H, W, _, _, deg, debug = b.geometry
    S, P = b.scenes, int(b.means.shape[-2])
    n, M = int(idx.numel()), int(shs_c.shape[1])
    counts = [n] if counts is None else counts
    V, n_max = st.nviews, max(counts)
    color = torch.empty((V, 3, H, W), dtype=torch.float32, device=dev)
    allmap = torch.empty((V, 8, H, W), dtype=torch.float32, device=dev)
    radii = torch.empty((V, n_max), dtype=torch.int32, device=dev)
    counts_coarse = st.resolve()    # capacity verified (stage 2 re-run if it overflowed) before the lists are read
    capacity = st.capacity
    geom_b, tile_b, image_b, _, pl_b = R._views_sizes(lib, V, n_max, H, W, capacity, for_backward)[:5]
    blob = R._blob(geom_b + tile_b + image_b, dev)
    geom, tile = blob[:geom_b], blob[geom_b:geom_b + tile_b]
    image = blob[geom_b + tile_b:] if for_backward else None
    point_list = R._blob(pl_b, dev)
    _lib.launch(
        "srf_scenes_subset_forward", dev, S, V // S, P, n, n_max, int(deg), M, _ptr(idx), _ptr(offsets),
        b.means.data_ptr(), _ptr(shs_c), None, b.cams.data_ptr(), H, W, capacity, b.radii.data_ptr(),
        st.geom.data_ptr(), st.tile.data_ptr(), _ptr(st.point_list), capacity, 1 if st.for_backward else 0,
        radii.data_ptr(), geom.data_ptr(), tile.data_ptr(), point_list.data_ptr(), _ptr(image), color.data_ptr(),
        allmap.data_ptr(), R._blob(_lib.subset_workspace_bytes(lib, S * P), dev).data_ptr(), 1 if for_backward else 0)
    Vs = V // S
    for s, c in enumerate(counts):
        if c == 0:      # a scene with an empty mask renders what a forward of zero Gaussians renders: zeros
            color[s * Vs:(s + 1) * Vs].zero_()
            allmap[s * Vs:(s + 1) * Vs].zero_()
    # the kept entries sit at the coarse list positions: the list's extent is the coarse one
    state = R.ForwardState(geom, tile, image, point_list if for_backward else None, capacity, counts_coarse, nviews=V,
                           cams=b.cams, for_backward=for_backward)
    if debug:
        torch.cuda.synchronize(dev)
    return ((*_epilogue_forward(color, allmap, b.rays, b.cams, b.depth_ratio), radii), (color, allmap, state))


class _RenderSubsetViews(torch.autograd.Function):
    """Inputs: the coarse centers, opacity, scales and rotations as the coarse render took them (S*P rows) and the
    concatenated ``shs_fine``; the gradients of the coarse tensors are the subsets' in their rows and zero elsewhere."""

    @staticmethod
    def forward(ctx, binning, nz, idx, offsets, counts, shs_c, centers, opacity, scales, rotations):
        outs, (color, allmap, state) = _subset_forward(binning, idx, shs_c, True, offsets, counts)
        radii = outs[-1]
        ctx.save_for_backward(nz, idx, offsets, shs_c, centers, scales, rotations, color, allmap, radii, state.geom,
                              state.tile, state.image)
        ctx.binning, ctx.state, ctx.n_max, ctx.opac_shape = binning, state, max(counts), tuple(opacity.shape)
        ctx.mark_non_differentiable(radii)
        return outs

    @staticmethod
    def backward(ctx, g_image, g_depth, g_acc, g_rn, g_dn, g_dist, _g_radii):
        nz, idx, offsets, shs, centers, scales, rotations, color, allmap, radii, _geom, _tile, _image = ctx.saved_tensors
        b = ctx.binning
        H, W, tfx, tfy, deg, debug = b.geometry
        P = int(b.means.shape[-2])
        SP = b.scenes * P
        d_color, d_allmap = _epilogue_backward(color, allmap, b.rays, b.cams, b.depth_ratio, b.rays is not None,
                                               g_image, g_depth, g_acc, g_rn, g_dn, g_dist)
        # the per-Gaussian backward reads the n subset rows of the flattened [S*P] coarse tensors (a gather, exact):
        # scene s's local index + s*P; its gradients go back to those rows
        rows_idx = nz[:, 0] * P + idx
        rows = [t.reshape(SP, -1).index_select(0, rows_idx).contiguous() for t in (centers, scales, rotations)]
        g = R.backward_batch_raw(ctx.state, radii, rows[0], shs, rows[1], rows[2], b.cams, list(zip(tfx, tfy)), H, W,
                                 deg, d_color, d_allmap, offsets=offsets, P=ctx.n_max, raw_activations=b.raw_activations, debug=debug)

        def scatter(gn, shape):
            full = torch.zeros(shape, dtype=torch.float32, device=idx.device)
            if idx.numel():
                full.view(SP, -1)[rows_idx] = gn.reshape(idx.numel(), -1)     # unique rows: an exact copy per row
            return full
        return (None, None, None, None, None, g["sh"], scatter(g["means3D"], tuple(centers.shape)),
                scatter(g["opacities"], ctx.opac_shape), scatter(g["scales"], tuple(scales.shape)),
                scatter(g["rotations"], tuple(rotations.shape)))


_F32_RATIO_LOW, _F32_RATIO_HIGH = np.float32(1e-3), np.float32(0.5)     # LaRa's thresholds as torch compares them


class FineSubset:
    """One compaction of the fine pass's masks [B,P] bool, shared by the point features, the fine head and the subset
    render: ``counts`` (host list, one read of ``masks.sum(1)``), ``offsets`` (host list [B+1]), ``offsets_d`` (the same
    on the device, int64, None for B = 1), ``nz`` the (scene, index) pairs [n,2] scene-major and ascending within a
    scene, ``idx`` their indices and ``rows`` the global rows b*P + index as int32.  ``masks`` are the masks the subset
    was built from.

    ``check=True`` first applies LaRa's ``Network._check_mask`` (lightning/network.py:381-388) to each scene in scene
    order, with the same ``torch.rand`` draws where LaRa draws, so that under one seed the masks are LaRa's bit for bit:
    the ratio is fp32(count) / fp32(P) compared with 1e-3 and 0.5 in fp32, as torch computes ``torch.sum(mask) /
    np.prod(mask.shape)``; a sparse scene becomes ``(mask + r) > 0.8`` and, with ``training``, a dense one
    ``(mask * r) > 0.5``.  The counts are read a second time only if some scene took a branch."""
    __slots__ = ("masks", "counts", "offsets", "offsets_d", "nz", "idx", "rows", "scenes", "P", "n")

    def __init__(self, masks: torch.Tensor, check: bool = False, training: bool = False):
        if not isinstance(masks, torch.Tensor) or masks.dtype != torch.bool or masks.ndim != 2:
            raise RuntimeError(f"FineSubset: masks must be a bool tensor [B,P], got {getattr(masks, 'dtype', type(masks))} "
                               f"{tuple(getattr(masks, 'shape', ()))}")
        B, P = (int(x) for x in masks.shape)
        if B < 1:
            raise RuntimeError("FineSubset: masks must hold at least one scene")
        if B * P >= 2 ** 31:
            raise RuntimeError(f"FineSubset: B*P = {B * P} rows are over the int32 index range")
        counts_d = masks.sum(1)
        counts = [int(c) for c in counts_d.tolist()]          # the host read
        if check:
            checked, changed = [], False
            for b, c in enumerate(counts):
                mask = masks[b]
                ratio = np.float32(c) / np.float32(P) if P else np.float32(np.nan)
                if ratio < _F32_RATIO_LOW:
                    mask = mask + torch.rand(mask.shape, device=mask.device) > 0.8
                    changed = True
                elif ratio > _F32_RATIO_HIGH and training:
                    mask = mask * torch.rand(mask.shape, device=mask.device) > 0.5
                    changed = True
                checked.append(mask)
            if changed:
                masks = torch.stack(checked)
                counts_d = masks.sum(1)
                counts = [int(c) for c in counts_d.tolist()]      # the second host read
        n = sum(counts)
        self.masks, self.counts, self.scenes, self.P, self.n = masks, counts, B, P, n
        self.offsets = [0]
        for c in counts:
            self.offsets.append(self.offsets[-1] + c)
        self.nz = torch.nonzero_static(masks, size=n)        # (scene, index) pairs, scene-major, ascending in a scene
        self.idx = self.nz[:, 1].contiguous()
        self.rows = (self.nz[:, 0] * P + self.nz[:, 1]).to(torch.int32)
        self.offsets_d = None      # one scene: the subset render takes idx[0..n) without offsets and waits for nothing
        if B > 1:
            self.offsets_d = torch.zeros(B + 1, dtype=torch.int64, device=masks.device)
            torch.cumsum(counts_d, 0, out=self.offsets_d[1:])


def _render_subset(fn, binning: SceneBinning, subset: FineSubset, shs_fine):
    """The subset render of every scene of ``binning`` (checked, unchanged) with the :class:`FineSubset` of its masks
    and ``shs_fine`` [n,M,3]; ``fn`` names the caller in messages.  Returns the outputs of :func:`_subset_forward`."""
    centers, _, opacity, scales, rotations = binning.tensors
    dev = binning.means.device
    deg = binning.geometry[4]
    if not isinstance(shs_fine, torch.Tensor) or shs_fine.dtype != torch.float32 or shs_fine.device != dev or \
            shs_fine.ndim != 3 or shs_fine.shape[2] != 3 or shs_fine.shape[1] < (deg + 1) ** 2:
        raise RuntimeError(f"{fn}: shs_fine must be float32 [n, M >= {(deg + 1) ** 2}, 3] on {dev}, got "
                           f"{getattr(shs_fine, 'dtype', type(shs_fine))} {tuple(getattr(shs_fine, 'shape', ()))}")
    counts, n = subset.counts, subset.n
    if shs_fine.shape[0] != n:
        raise RuntimeError(f"{fn}: shs_fine has {shs_fine.shape[0]} rows, the mask selects {n}")
    nz, idx, offsets = subset.nz, subset.idx, subset.offsets_d
    shs_c = shs_fine.contiguous()
    with _DeviceGuard(dev):
        if R.needs_backward(centers, shs_fine, opacity, scales, rotations):
            outs = _RenderSubsetViews.apply(binning, nz, idx, offsets, counts, shs_c, centers, opacity, scales, rotations)
        else:
            outs = _subset_forward(binning, idx, shs_c, False, offsets, counts)[0]
    return outs


def render_subset_views(binning: SceneBinning, mask: torch.Tensor, shs_fine: torch.Tensor,
                        prex: str = "_fine") -> Dict[str, torch.Tensor]:
    """LaRa's fine-pass render (network.py:486-525 with ``_centers[mask]``, ``_opacity_coarse[i][mask]``, ...) from the
    coarse pass's binning: ``binning`` is ``out["binning"]`` of ``render_scene_views(..., keep_binning=True)``, ``mask``
    a bool tensor [P] on the Gaussians' device, ``shs_fine`` the subset's SH coefficients [n, M, 3].  Returns the dict
    ``render_scene_views`` returns for the gathered subset (same keys, layout and bits, ``radii`` [V, n]) without a
    preprocess, scatter or sort: the coarse records are copied with a new colour and the coarse tile lists filtered to
    the mask.  One host sync (the mask count).  The gradients of the coarse centers, opacity, scales and
    rotations are those of the gathered path; under ``no_grad`` / ``inference_mode`` the forward-only path is taken."""
    if not isinstance(binning, SceneBinning) or binning.scenes != 1:
        raise TypeError("render_subset_views: binning must be out['binning'] of render_scene_views(..., keep_binning=True)")
    binning.check_unchanged()
    P, dev = int(binning.means.shape[-2]), binning.means.device
    if not isinstance(mask, torch.Tensor) or mask.dtype != torch.bool or tuple(mask.shape) != (P,) or mask.device != dev:
        raise RuntimeError(f"render_subset_views: mask must be a bool tensor [{P}] on {dev}, got "
                           f"{getattr(mask, 'dtype', type(mask))} {tuple(getattr(mask, 'shape', ()))} on "
                           f"{getattr(mask, 'device', None)}")
    outs = _render_subset("render_subset_views", binning, FineSubset(mask[None]), shs_fine)
    return _out_dict(*outs, binning.rays is not None, prex)


def concat_views(out: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """The layout LaRa's step hands to the loss: ``torch.cat([frame[k] for frame in views], dim=1)``
    (network.py:525), i.e. the views side by side along the width."""
    res = {}
    for k, t in out.items():
        if k.startswith("radii") or not isinstance(t, torch.Tensor):     # radii, the kept binning
            continue
        if t.ndim == 4:      # [V,H,W,C] -> [H, V*W, C]
            V, H, W, C = t.shape
            res[k] = t.permute(1, 0, 2, 3).reshape(H, V * W, C)
        else:                # [V,H,W] -> [H, V*W]
            V, H, W = t.shape
            res[k] = t.permute(1, 0, 2).reshape(H, V * W)
    return res


# ---------------------------------------------------------------------------------------------------------------------
# B scenes in one launch set (srf_scenes_*, DESIGN §3.21): the B*V views of a batch are rendered as one V-view call
# whose preprocess and per-Gaussian backward read each view's Gaussians from its own scene.
# ---------------------------------------------------------------------------------------------------------------------

def batch_view_settings(settings: Sequence[Sequence[R.GaussianRasterizationSettings]]):
    """(H, W, [(tanfovx, tanfovy)] per scene, sh_degree, prefiltered, debug) of a batch: each scene's views share what
    :func:`shared_view_settings` requires, and all scenes share V, the image size and the SH degree."""
    if len(settings) == 0 or any(len(s) == 0 for s in settings):
        raise ValueError("render_batch_views needs at least one scene of at least one view")
    V = len(settings[0])
    keys = [shared_view_settings(list(s)) for s in settings]
    for s, k in zip(settings, keys):
        if len(s) != V:
            raise RuntimeError("render_batch_views: all scenes of a batch must have the same number of views")
        if (k[0], k[1], k[4]) != (keys[0][0], keys[0][1], keys[0][4]):
            raise RuntimeError("render_batch_views: all scenes of a batch must share the image size and the SH degree")
    return (keys[0][0], keys[0][1], [(k[2], k[3]) for k in keys], keys[0][4], any(k[5] for k in keys),
            any(k[6] for k in keys))


def _batch_inputs(centers, shs, opacity, scales, rotations):
    """Shape checks of the [B,P,...] Gaussian tensors; returns them fp32 contiguous, opacity as [B,P]."""
    if not isinstance(centers, torch.Tensor) or centers.ndim != 3 or centers.shape[2] != 3:
        raise RuntimeError("render_batch_views: centers must be [B,P,3]")
    B, P = int(centers.shape[0]), int(centers.shape[1])
    want = {"shs": (shs, 4), "scales": (scales, 3), "rotations": (rotations, 3)}
    for name, (t, nd) in want.items():
        if not isinstance(t, torch.Tensor) or t.ndim != nd or tuple(t.shape[:2]) != (B, P):
            raise RuntimeError(f"render_batch_views: {name} must be [B,P,...] = [{B},{P},...]")
    if shs.shape[3] != 3 or scales.shape[2] != 2 or rotations.shape[2] != 4:
        raise RuntimeError("render_batch_views: shs must be [B,P,M,3], scales [B,P,2] and rotations [B,P,4]")
    if not isinstance(opacity, torch.Tensor) or opacity.numel() != B * P or tuple(opacity.shape[:2]) != (B, P):
        raise RuntimeError(f"render_batch_views: opacity must be [B,P] or [B,P,1] = [{B},{P}]")
    return tuple(R._f32c(t, n) for t, n in ((centers, "centers"), (shs, "shs"), (opacity.reshape(B, P), "opacity"),
                                            (scales, "scales"), (rotations, "rotations")))


def _batch_out_dict(outs, B, has_rays, prex):
    """{key: [B,V,...]} of the [B*V,...] outputs, the layout of :func:`render_scene_views` per scene."""
    out = _out_dict(*outs, has_rays, prex)
    return {k: t.view((B, t.shape[0] // B) + tuple(t.shape[1:])) for k, t in out.items()}


class BatchCameras(NamedTuple):
    """The cameras of a batch as records: ``cams`` f32 [B*V, SRF_CAM_FLOATS] on the Gaussians' device (scene b's views
    are rows b*V .. b*V+V-1; ``lara_b200.batch.batch_cameras`` builds them), the image size ``H``, ``W``, ``tan_fov``
    one pair (tan_fovx, tan_fovy) of finite positive values per scene, and ``sh_degree``."""
    cams: torch.Tensor
    H: int
    W: int
    tan_fov: Sequence
    sh_degree: int


def _batch_cameras(cameras: BatchCameras, dev, B):
    """(cams, H, W, tan_fov, sh_degree, prefiltered, debug) of checked :class:`BatchCameras` for B scenes."""
    fn = "render_batch_views"
    cams, H, W, tan_fov, deg = cameras
    tan_fov = [(float(x), float(y)) for x, y in tan_fov]
    if len(tan_fov) != B:
        raise RuntimeError(f"{fn}: cameras.tan_fov must hold one pair per scene ({B}), got {len(tan_fov)}")
    if not all(0.0 < t < float("inf") for p in tan_fov for t in p):
        raise RuntimeError(f"{fn}: cameras.tan_fov must be finite and positive, got {tan_fov}")
    if not isinstance(cams, torch.Tensor) or cams.dtype != torch.float32 or cams.ndim != 2 or \
            cams.shape[1] != _lib.CAM_FLOATS or cams.shape[0] % B != 0 or cams.shape[0] == 0 or cams.device != dev:
        raise RuntimeError(f"{fn}: cameras.cams must be float32 [B*V,{_lib.CAM_FLOATS}] with B = {B} on {dev}, got "
                           f"{getattr(cams, 'dtype', type(cams))} {tuple(getattr(cams, 'shape', ()))} on "
                           f"{getattr(cams, 'device', None)}")
    if int(H) < 1 or int(W) < 1 or not 0 <= int(deg) <= 3:
        raise RuntimeError(f"{fn}: cameras need H, W >= 1 and sh_degree in [0, 3], got {H}, {W}, {deg}")
    return cams.detach().contiguous(), int(H), int(W), tan_fov, int(deg), False, False


def render_batch_views(centers, shs, opacity, scales, rotations,
                       settings: Optional[Sequence[Sequence[R.GaussianRasterizationSettings]]] = None,
                       rays: Optional[torch.Tensor] = None, depth_ratio: float = 0.0, raw_activations: bool = False,
                       prex: str = "", keep_binning: bool = False,
                       cameras: Optional[BatchCameras] = None) -> Dict[str, object]:
    """All views of all B scenes of a batch in one autograd node and one launch set: ``centers`` [B,P,3], ``shs``
    [B,P,M,3], ``opacity`` [B,P] or [B,P,1], ``scales`` [B,P,2], ``rotations`` [B,P,4], ``settings[b]`` scene b's V
    view settings, ``rays`` [B,V,H,W,6] or None.  Returns ``{key+prex: [B,V,...]}``, where ``out[k][b]`` is what
    :func:`render_scene_views` returns for scene b alone (bit for bit), and ``radii+prex`` [B,V,P].  Scenes may differ
    in field of view and background; they must share V, the image size and the SH degree.  No-grad renders take the
    forward-only path.  ``keep_binning=True`` adds ``out["binning"+prex]``, a :class:`SceneBinning` of B scenes for
    :func:`render_batch_subset_views`.

    ``cameras`` (a :class:`BatchCameras`, in place of ``settings``) gives the views as camera records already on the
    device, so that no per-view settings object is built; the records of ``pack_cameras`` over ``settings`` render
    the same bits."""
    dev = centers.device
    inputs = _batch_inputs(centers, shs, opacity, scales, rotations)
    if (settings is None) == (cameras is None):
        raise TypeError("render_batch_views: pass either settings or cameras")
    if cameras is None:
        settings = [[R._check_settings(rs, dev) for rs in s] for s in settings]
        H, W, tan_fov, deg, prefiltered, debug = batch_view_settings(settings)
        B, V = len(settings), len(settings[0])
        cams = _pack([rs for s in settings for rs in s], dev)
    else:
        B = int(centers.shape[0])
        cams, H, W, tan_fov, deg, prefiltered, debug = _batch_cameras(cameras, dev, B)
        V = int(cams.shape[0]) // B
    rays_c = None
    if rays is not None:
        rays_c = rays.contiguous()
        if rays_c.dtype != torch.float32 or tuple(rays_c.shape) != (B, V, H, W, 6) or rays_c.device != dev:
            raise RuntimeError(f"rays must be float32 [B,V,H,W,6] = {(B, V, H, W, 6)} on {dev}, got "
                               f"{rays_c.dtype} {tuple(rays_c.shape)} on {rays_c.device}")
        rays_c = rays_c.view(B * V, H, W, 6)
    tfx, tfy = zip(*tan_fov)
    outs, binning = _render_views(inputs, rays_c, cams, (H, W, tfx, tfy, deg, debug),
                                  prefiltered, float(depth_ratio), bool(raw_activations), keep_binning,
                                  (centers, shs, opacity, scales, rotations))
    out = _batch_out_dict(outs, B, rays is not None, prex)
    if binning is not None:
        out["binning" + prex] = binning
    return out


def render_batch_subset_views(binning: SceneBinning, masks, shs_fine: torch.Tensor,
                              prex: str = "_fine") -> Dict[str, object]:
    """LaRa's fine pass for all B scenes of a batch from the coarse pass's binning: ``binning`` is ``out["binning"]`` of
    ``render_batch_views(..., keep_binning=True)``, ``masks`` a bool tensor [B,P] or the :class:`FineSubset` of those
    masks (whose counts are then not read again), ``shs_fine`` [n,M,3] the subsets' SH coefficients concatenated in scene
    order (``FineHead.fine_shs``' batch form, or B of its calls concatenated).  Returns ``{key+prex: [B,V,...]}`` where
    ``out[k][b]`` is what :func:`render_subset_views` returns for scene b alone, bit for bit, and ``radii+prex`` a list of
    B tensors [V, n_b].  One host sync for the mask counts when given masks (and, for B > 1, the C entry's check of the
    offsets, which waits for the stream).  Gradients go to the [B,P,...] coarse tensors and to ``shs_fine``."""
    fn = "render_batch_subset_views"
    if not isinstance(binning, SceneBinning):
        raise TypeError("render_batch_subset_views: binning must be out['binning'] of render_batch_views(..., "
                        "keep_binning=True)")
    binning.check_unchanged()
    B, P, dev = binning.scenes, int(binning.means.shape[-2]), binning.means.device
    given = masks.masks if isinstance(masks, FineSubset) else masks
    if not isinstance(given, torch.Tensor) or given.dtype != torch.bool or tuple(given.shape) != (B, P) or \
            given.device != dev:
        raise RuntimeError(f"{fn}: masks must be a bool tensor [{B},{P}] on {dev} or its FineSubset, got "
                           f"{getattr(given, 'dtype', type(given))} {tuple(getattr(given, 'shape', ()))} on "
                           f"{getattr(given, 'device', None)}")
    subset = masks if isinstance(masks, FineSubset) else FineSubset(masks)
    outs = _render_subset(fn, binning, subset, shs_fine)
    radii = outs[-1]
    out = _batch_out_dict(outs, B, binning.rays is not None, prex)
    V = radii.shape[0] // B
    out["radii" + prex] = [radii[b * V:(b + 1) * V, :subset.counts[b]] for b in range(B)]
    return out
