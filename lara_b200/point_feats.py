"""Fused point-feature sampler of LaRa's fine pass (``Network.get_point_feats``, lightning/network.py:390-411, with
``projection`` at :182-187) -- an additional entry point next to the unchanged rasterizer.

``sample_point_feats(points, img_ref, renderings, src_w2cs, src_ixts)`` returns exactly what ``get_point_feats``
returns for ``points[mask]``: the ``[V, 8, n]`` features img_ref (3) | image (3) | acc_map (1) | |depth - z| (1),
bilinearly sampled at each point's projection into the V source views.  One CUDA kernel per direction replaces the
bmm projections, the two concatenations of the image stacks, ``grid_sample`` and its backward (which forms, and drops,
a gradient for the constant source image too) and the slice / abs / cat ops.  A maintainer switches LaRa to it with::

    def get_point_feats(self, idx, img_ref, renderings, n_views_sel, batch, points, mask):
        return sample_point_feats(points[mask], img_ref, renderings,
                                  batch['tar_w2c'][idx, :n_views_sel], batch['tar_ixt'][idx, :n_views_sel]), mask

The rendering tensors are read in planar layout: ``permute(0, 3, 1, 2)`` of the channel-last views
``render_scene_views`` returns is its epilogue's own ``[V, C, H, W]`` buffer, so for those no copy is made.  Their
gradients come back through the same permutes and add to the loss gradients of the coarse outputs.

Differences from the reference, by design: a sample coordinate that is not finite (a point in a source camera's
plane, z = 0) samples 0 and passes no gradient through the grid; ``img_ref``, ``src_w2cs`` and ``src_ixts`` are
constants (passing one that requires grad raises); under autocast the projection runs in fp32, where LaRa's matmuls
would run in bf16.
"""
from __future__ import annotations

import ctypes
from typing import Dict

import torch

from . import _lib
from ._lib import _ptr


_NAMES = ("points", "img_ref", "renderings['image']", "renderings['acc_map']", "renderings['depth']", "src_w2cs",
          "src_ixts")


def _check_shapes(points, img_ref, image, acc, depth, w2cs, ixts):
    """Shape checks on the caller's tensors (renderings channel-last); returns (V, H, W)."""
    for name, t in zip(_NAMES, (points, img_ref, image, acc, depth, w2cs, ixts)):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"sample_point_feats: {name} must be a tensor")
    if points.ndim != 2 or points.shape[1] != 3:
        raise RuntimeError(f"sample_point_feats: points must be [n,3], got {tuple(points.shape)}")
    if img_ref.ndim != 4 or img_ref.shape[1] != 3:
        raise RuntimeError(f"sample_point_feats: img_ref must be [V,3,H,W], got {tuple(img_ref.shape)}")
    V, _, H, W = (int(s) for s in img_ref.shape)
    for name, t, shape in zip(_NAMES[2:], (image, acc, depth, w2cs, ixts),
                              ((V, H, W, 3), (V, H, W), (V, H, W, 1), (V, 4, 4), (V, 3, 3))):
        if tuple(t.shape) != shape:
            raise RuntimeError(f"sample_point_feats: {name} must be {shape}, got {tuple(t.shape)}")
    return V, H, W


def _check_tensors(tensors):
    """dtype / device / constant checks before any launch: the kernels take raw pointers and do not differentiate
    img_ref or the cameras."""
    for name, t in zip(_NAMES, tensors):
        if name in ("img_ref", "src_w2cs", "src_ixts") and t.requires_grad:
            raise RuntimeError(f"sample_point_feats: {name} requires grad, but the sampler treats it as a constant "
                               "(as LaRa does); detach it")
    dev = tensors[0].device
    for name, t in zip(_NAMES, tensors):
        if t.dtype != torch.float32:
            raise RuntimeError(f"sample_point_feats: expected scalar type Float but found {t.dtype} for {name}")
        if not t.is_cuda or t.device != dev:
            raise RuntimeError(f"sample_point_feats: {name} must be a CUDA tensor on {dev}, got {t.device}")


class _PointFeats(torch.autograd.Function):
    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, points, img_ref, image, acc, depth, w2cs, ixts):
        _check_tensors((points, img_ref, image, acc, depth, w2cs, ixts))
        V, _, H, W = (int(s) for s in img_ref.shape)
        ins = [t.contiguous() for t in (points, w2cs, ixts, img_ref, image, acc, depth)]
        n = int(points.shape[0])
        feats = torch.empty((V, 8, n), dtype=torch.float32, device=points.device)
        _lib.launch("srf_point_feats_forward", points.device, V, n, H, W, *[t.data_ptr() for t in ins],
                    feats.data_ptr())
        ctx.save_for_backward(*ins)
        ctx.dims = (V, n, H, W)
        return feats

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, g_feats):
        ins = ctx.saved_tensors
        V, n, H, W = ctx.dims
        dev = g_feats.device
        need = ctx.needs_input_grad

        def new(wanted, *shape):
            return torch.empty(shape, dtype=torch.float32, device=dev) if wanted else None
        g_points, g_image, g_acc, g_depth = new(need[0], n, 3), new(need[2], V, 3, H, W), new(need[3], V, H, W), \
            new(need[4], V, 1, H, W)
        g_feats = g_feats.contiguous()
        # fixed-point sums in a workspace instead of atomics
        ws = (torch.empty(_lib.det_point_feats_workspace_bytes(_lib.load(), V, H, W), dtype=torch.uint8, device=dev)
              if _lib.deterministic() else None)
        _lib.launch("srf_point_feats_backward", dev, V, n, H, W, *[t.data_ptr() for t in ins], g_feats.data_ptr(),
                    _ptr(g_points), _ptr(g_image), _ptr(g_acc), _ptr(g_depth), _ptr(ws))
        return g_points, None, g_image, g_acc, g_depth, None, None


def sample_point_feats(points: torch.Tensor, img_ref: torch.Tensor, renderings: Dict[str, torch.Tensor],
                       src_w2cs: torch.Tensor, src_ixts: torch.Tensor) -> torch.Tensor:
    """``[V, 8, n]`` point features of ``get_point_feats`` (network.py:390-411) for the points ``[n, 3]``.

    ``img_ref`` [V,3,H,W] is the source images; ``renderings`` holds the coarse pass's ``image`` [V,H,W,3],
    ``acc_map`` [V,H,W] and ``depth`` [V,H,W,1] of the same V views (e.g. ``render_scene_views``'s dict sliced to the
    first V views); ``src_w2cs`` [V,4,4] and ``src_ixts`` [V,3,3] are the views' row-major world-to-camera and
    intrinsic matrices.  Differentiable wrt ``points`` and the three renderings."""
    for k in ("image", "acc_map", "depth"):
        if k not in renderings:
            raise KeyError(f"sample_point_feats: renderings has no '{k}'")
    image, acc, depth = renderings["image"], renderings["acc_map"], renderings["depth"]
    _check_shapes(points, img_ref, image, acc, depth, src_w2cs, src_ixts)
    return _PointFeats.apply(points, img_ref, image.permute(0, 3, 1, 2), acc, depth.permute(0, 3, 1, 2),
                             src_w2cs, src_ixts)


_BATCH_NAMES = ("centers", "img_ref", "renderings['image']", "renderings['acc_map']", "renderings['depth']", "w2cs",
                "ixts")


class _BatchPointFeats(torch.autograd.Function):
    """(subset, centers [B,P,3], img_ref [B,Vs,3,H,W], image [B,V,3,H,W], acc [B,V,H,W], depth [B,V,1,H,W], w2cs, ixts)
    -> feats [Vs,8,n]; the rendering gradients are the full [B,V,...] planes (0 for views >= Vs)."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, subset, centers, img_ref, image, acc, depth, w2cs, ixts):
        fn = "sample_batch_point_feats"
        named = list(zip(_BATCH_NAMES, (centers, img_ref, image, acc, depth, w2cs, ixts)))
        _check_tensors_named(fn, named)
        B, P = int(centers.shape[0]), int(centers.shape[1])
        Vs, _, H, W = (int(s) for s in img_ref.shape[1:])
        V = int(image.shape[1])
        ins = [t.contiguous() for t in (centers, w2cs, ixts, image, acc, depth)]
        n = subset.n
        feats = torch.empty((Vs, 8, n), dtype=torch.float32, device=centers.device)
        offsets = (ctypes.c_int64 * (B + 1))(*subset.offsets)
        addr = _lib.PfImageAddr(*(int(s) for s in img_ref.stride()))
        args = (B, Vs, V, P, n, H, W, offsets, subset.rows.data_ptr(), *[t.data_ptr() for t in ins[:3]],
                img_ref.data_ptr(), ctypes.byref(addr), *[t.data_ptr() for t in ins[3:]])
        _lib.launch("srf_point_feats_scenes_forward", centers.device, *args, feats.data_ptr())
        ctx.save_for_backward(subset.rows, img_ref, *ins)
        ctx.dims = (B, Vs, V, P, n, H, W, list(subset.offsets))
        return feats

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, g_feats):
        rows, img_ref, centers, w2cs, ixts, image, acc, depth = ctx.saved_tensors
        B, Vs, V, P, n, H, W, offs = ctx.dims
        dev = g_feats.device
        need = ctx.needs_input_grad

        def new(wanted, *shape):
            return torch.empty(shape, dtype=torch.float32, device=dev) if wanted else None
        g_centers, g_image, g_acc, g_depth = (new(need[1], B, P, 3), new(need[3], B, V, 3, H, W),
                                              new(need[4], B, V, H, W), new(need[5], B, V, 1, H, W))
        g_feats = g_feats.contiguous()
        # fixed-point sums in a workspace instead of atomics, one scale per scene
        ws = (torch.empty(_lib.det_point_feats_scenes_workspace_bytes(_lib.load(), B, Vs, H, W), dtype=torch.uint8,
                          device=dev) if _lib.deterministic() else None)
        offsets = (ctypes.c_int64 * (B + 1))(*offs)
        addr = _lib.PfImageAddr(*(int(s) for s in img_ref.stride()))
        _lib.launch("srf_point_feats_scenes_backward", dev, B, Vs, V, P, n, H, W, offsets, rows.data_ptr(),
                    centers.data_ptr(), w2cs.data_ptr(), ixts.data_ptr(), img_ref.data_ptr(), ctypes.byref(addr),
                    image.data_ptr(), acc.data_ptr(), depth.data_ptr(), g_feats.data_ptr(), _ptr(g_centers),
                    _ptr(g_image), _ptr(g_acc), _ptr(g_depth), _ptr(ws))
        return None, g_centers, None, g_image, g_acc, g_depth, None, None


def _check_tensors_named(fn, named):
    """dtype / device / constant checks of ``(name, tensor)`` pairs before any launch."""
    for name, t in named:
        if name in ("img_ref", "w2cs", "ixts") and t.requires_grad:
            raise RuntimeError(f"{fn}: {name} requires grad, but the sampler treats it as a constant (as LaRa does); "
                               "detach it")
    dev = named[0][1].device
    for name, t in named:
        if t.dtype != torch.float32:
            raise RuntimeError(f"{fn}: expected scalar type Float but found {t.dtype} for {name}")
        if not t.is_cuda or t.device != dev:
            raise RuntimeError(f"{fn}: {name} must be a CUDA tensor on {dev}, got {t.device}")


def sample_batch_point_feats(subset, centers: torch.Tensor, img_ref: torch.Tensor, renderings: Dict[str, torch.Tensor],
                             w2cs: torch.Tensor, ixts: torch.Tensor) -> torch.Tensor:
    """:func:`sample_point_feats` for all B scenes of a batch in one launch per direction: ``[Vs, 8, n]``, scene b's
    points (``subset``'s rows of scene b, in order) at columns ``subset.offsets[b] .. subset.offsets[b+1]``, each column
    bit for bit what ``sample_point_feats(centers[b][mask_b], ...)`` returns.

    ``subset`` is the :class:`lara_b200.multiview.FineSubset` of the masks [B,P]; ``centers`` [B,P,3] the coarse centres
    (the kernel gathers the subset itself); ``img_ref`` [B,Vs,3,H,W] the source images at any strides (LaRa's ``_inps``
    or a channel-last ``tar_rgb[:, :Vs]`` view are read in place); ``renderings`` :func:`render_batch_views`' dict,
    ``image`` [B,V,H,W,3], ``acc_map`` [B,V,H,W], ``depth`` [B,V,H,W,1] with V >= Vs, read from the render's own planar
    buffers (scene b's first Vs views); ``w2cs`` [B,Vs,4,4], ``ixts`` [B,Vs,3,3].  Differentiable wrt ``centers`` and
    the three renderings: the centres' gradient is the subset rows' sum over the views and 0 elsewhere, the renderings'
    is 0 for views >= Vs.  ``img_ref`` and the cameras are constants.  Under autocast it computes in fp32."""
    from .multiview import FineSubset
    fn = "sample_batch_point_feats"
    if not isinstance(subset, FineSubset):
        raise TypeError(f"{fn}: subset must be a lara_b200.multiview.FineSubset, got {type(subset).__name__}")
    for k in ("image", "acc_map", "depth"):
        if k not in renderings:
            raise KeyError(f"{fn}: renderings has no '{k}'")
    image, acc, depth = renderings["image"], renderings["acc_map"], renderings["depth"]
    for name, t in zip(_BATCH_NAMES, (centers, img_ref, image, acc, depth, w2cs, ixts)):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{fn}: {name} must be a tensor")
    B, P = subset.scenes, subset.P
    if tuple(centers.shape) != (B, P, 3):
        raise RuntimeError(f"{fn}: centers must be [B,P,3] = {(B, P, 3)} (the subset's), got {tuple(centers.shape)}")
    if img_ref.ndim != 5 or img_ref.shape[0] != B or img_ref.shape[2] != 3:
        raise RuntimeError(f"{fn}: img_ref must be [{B},Vs,3,H,W], got {tuple(img_ref.shape)}")
    Vs, _, H, W = (int(s) for s in img_ref.shape[1:])
    if image.ndim != 5 or tuple(image.shape[:1]) + tuple(image.shape[2:]) != (B, H, W, 3) or image.shape[1] < Vs:
        raise RuntimeError(f"{fn}: renderings['image'] must be [{B},V,{H},{W},3] with V >= {Vs}, got "
                           f"{tuple(image.shape)}")
    V = int(image.shape[1])
    for name, t, shape in zip(_BATCH_NAMES[3:], (acc, depth, w2cs, ixts),
                              ((B, V, H, W), (B, V, H, W, 1), (B, Vs, 4, 4), (B, Vs, 3, 3))):
        if tuple(t.shape) != shape:
            raise RuntimeError(f"{fn}: {name} must be {shape}, got {tuple(t.shape)}")
    if subset.masks.device != centers.device:
        raise RuntimeError(f"{fn}: the subset is on {subset.masks.device}, centers on {centers.device}")
    return _BatchPointFeats.apply(subset, centers, img_ref, image.permute(0, 1, 4, 2, 3), acc,
                                  depth.permute(0, 1, 4, 2, 3), w2cs, ixts)
