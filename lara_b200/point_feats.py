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

from typing import Dict

import torch

from . import _lib
from .rasterizer import _DeviceGuard, _raw_stream


def _p(t) -> int:
    return 0 if t is None else t.data_ptr()


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
        lib = _lib.load()
        ins = [t.contiguous() for t in (points, w2cs, ixts, img_ref, image, acc, depth)]
        n = int(points.shape[0])
        dev = points.device
        feats = torch.empty((V, 8, n), dtype=torch.float32, device=dev)
        with _DeviceGuard(dev):
            _lib.check(lib.srf_point_feats_forward(_raw_stream(dev), V, n, H, W, *[t.data_ptr() for t in ins],
                                                   feats.data_ptr()), lib)
        ctx.save_for_backward(*ins)
        ctx.dims = (V, n, H, W)
        return feats

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, g_feats):
        lib = _lib.load()
        ins = ctx.saved_tensors
        V, n, H, W = ctx.dims
        dev = g_feats.device
        need = ctx.needs_input_grad

        def new(wanted, *shape):
            return torch.empty(shape, dtype=torch.float32, device=dev) if wanted else None
        g_points, g_image, g_acc, g_depth = new(need[0], n, 3), new(need[2], V, 3, H, W), new(need[3], V, H, W), \
            new(need[4], V, 1, H, W)
        g_feats = g_feats.contiguous()
        with _DeviceGuard(dev):
            _lib.check(lib.srf_point_feats_backward(_raw_stream(dev), V, n, H, W, *[t.data_ptr() for t in ins],
                                                    g_feats.data_ptr(), _p(g_points), _p(g_image), _p(g_acc),
                                                    _p(g_depth)), lib)
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
