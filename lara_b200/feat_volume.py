"""Fused feature-volume lifting of LaRa's coarse pass (``Network.build_feat_vol``, lightning/network.py:352-379, the
view-embedding concatenation of :451-452 and the block layout of ``VolTransformer.forward``, :145-150) -- an
additional entry point next to the unchanged rasterizer.

``FeatVolume`` holds the parameters of that stage under LaRa's ``Network`` names (``dir_norm.norm``,
``dir_norm.mlp.1``, ``view_embed`` and the buffer ``volume_grid``), so ``load_state_dict(network.state_dict(),
strict=False)`` fills it, and ``fv.dir_norm = network.dir_norm`` shares LaRa's parameters without copying them.  Its
two entries run on the kernels of csrc/feat_volume.cu (include/surfel_feat_volume.h):

* ``fv(img_feats, rays_down, w2cs, ixts, image_hw) -> [B,V,C,R,R,R]`` is the drop-in for ``build_feat_vol``;
* ``fv.cond_tokens(img_feats, rays_down, w2cs, ixts, image_hw, n_group) -> [B g^3, V bs^3, C+E]`` also replaces the
  ``cat`` with ``view_embed`` and the ``unfold`` / ``einsum`` blocks ``VolTransformer.forward`` passes its layers.

The arguments are the tensors LaRa builds at network.py:355-365 and :445: ``img_feats [B V,C,h,w]``, ``rays_down
[B,V,h,w,6]``, ``w2cs [B,V,4,4]``, ``ixts [B,V,3,3]``, ``image_hw = src_inps.shape[-2:]``.  Autograd keeps only the
inputs; the backward recomputes the forward, uses no float atomics and is bit-reproducible with or without
``torch.use_deterministic_algorithms`` (DESIGN §3.17).

Differences from the reference, by design: a voxel whose sample coordinate is not finite (in a source camera's plane)
samples 0 and passes no gradient; ``rays_down``, ``w2cs`` and ``ixts`` are constants (passing one that requires grad
raises); the op always computes in fp32, where under bf16 autocast LaRa's ``Linear`` in ``dir_norm`` and its
projection matmuls run in bf16.
"""
from __future__ import annotations

import torch
from torch import nn

from . import _lib

SH_FEATURES = 32


def dense_grid(reso: int, scene_size: float = 0.5) -> torch.Tensor:
    """``Network.build_dense_grid``: voxel centres of a reso^3 grid over [-scene_size, scene_size]^3, 'ij' order."""
    a = torch.arange(reso)
    grid = torch.stack(torch.meshgrid(a, a, a, indexing="ij"), dim=-1)
    grid = (grid + 0.5) / reso * 2 - 1
    return grid.reshape(reso, reso, reso, 3) * scene_size


class ModLN(nn.Module):
    """LaRa's ``ModLN`` parameter holder (network.py:190-213): ``norm`` and ``mlp = Sequential(SiLU, Linear)``."""

    def __init__(self, inner_dim: int, mod_dim: int = SH_FEATURES, eps: float = 1e-6):
        super().__init__()
        self.norm = nn.LayerNorm(inner_dim, eps=eps)
        self.mlp = nn.Sequential(nn.SiLU(), nn.Linear(mod_dim, inner_dim * 2))


class _FeatVolume(torch.autograd.Function):
    """(img_feats, rays, w2cs, ixts, grid [R,R,R,3], view_embed [Vmax,E] or None, (H_img, W_img), n_group, norm w,
    norm b, mlp w, mlp b) -> the output in the layout n_group selects (0 = drop-in)."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, x, rays, w2cs, ixts, grid, ve, image_hw, n_group, *params):
        ins = [t.contiguous() for t in (x, rays, w2cs, ixts, grid)]
        params = [p.contiguous() for p in params]
        ve = ve.contiguous() if ve is not None else None
        B, V, h, w = (int(s) for s in rays.shape[:4])
        C, R = int(x.shape[1]), int(grid.shape[0])
        Vmax, E = (int(ve.shape[0]), int(ve.shape[1])) if ve is not None else (0, 0)
        dev = x.device
        dims = (B, V, C, h, w, R, E, Vmax, int(image_hw[0]), int(image_hw[1]), n_group)
        if n_group == 0:
            out = torch.empty((B, V, C, R, R, R), dtype=torch.float32, device=dev)
        else:
            bs = R // n_group
            out = torch.empty((B * n_group ** 3, V * bs ** 3, C + E), dtype=torch.float32, device=dev)
        ws = _workspace(dev, dims)
        _lib.launch("srf_feat_volume_forward", dev, *dims, *[t.data_ptr() for t in ins],
                    *[p.data_ptr() for p in params], ve.data_ptr() if ve is not None else None, ws.data_ptr(),
                    out.data_ptr())
        ctx.save_for_backward(*ins, *params)
        ctx.dims = dims
        ctx.ve_shape = None if ve is None else ve.shape
        return out

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, g):
        x, rays, w2cs, ixts, grid, *params = ctx.saved_tensors
        dims = ctx.dims
        dev = x.device
        g = g.contiguous()
        g_x = torch.empty_like(x)
        g_params = [torch.empty_like(p) for p in params]
        g_ve = torch.empty(ctx.ve_shape, dtype=torch.float32, device=dev) if ctx.ve_shape is not None else None
        ws = _workspace(dev, dims)
        _lib.launch("srf_feat_volume_backward", dev, *dims, x.data_ptr(), rays.data_ptr(), w2cs.data_ptr(),
                    ixts.data_ptr(), grid.data_ptr(), *[p.data_ptr() for p in params], g.data_ptr(), ws.data_ptr(),
                    g_x.data_ptr(), *[p.data_ptr() for p in g_params], g_ve.data_ptr() if g_ve is not None else None)
        return (g_x, None, None, None, None, g_ve, None, None, *g_params)


def _workspace(dev, dims):
    B, V, C, h, w, R, E = dims[:7]
    with _lib._DeviceGuard(dev):
        n = _lib.feat_volume_workspace_bytes(_lib.load(), B, V, C, h, w, R, E)
    return torch.empty(n, dtype=torch.uint8, device=dev)


class FeatVolume(nn.Module):
    """The feature-volume stage of LaRa's ``Network``: ``dir_norm`` (``ModLN(C, 32, eps=1e-6)``), ``view_embed``
    ``[1, n_views, E, 1, 1, 1]`` when ``view_embed_dim`` > 0, and the buffer ``volume_grid [R,R,R,3]``, with LaRa's
    names, shapes and initialisation."""

    def __init__(self, feat_dim: int = 768, view_embed_dim: int = 32, feat_vol_reso: int = 16, n_views: int = 4,
                 scene_size: float = 0.5):
        super().__init__()
        if feat_dim % 32 != 0 or not 32 <= feat_dim <= 1024:
            raise ValueError(f"FeatVolume: feat_dim must be a multiple of 32 up to 1024, got {feat_dim}")
        if not 0 <= view_embed_dim <= 128:
            raise ValueError(f"FeatVolume: view_embed_dim must be in [0, 128], got {view_embed_dim}")
        if not 1 <= feat_vol_reso <= 64:
            raise ValueError(f"FeatVolume: feat_vol_reso must be in [1, 64], got {feat_vol_reso}")
        if view_embed_dim > 0 and n_views < 1:
            raise ValueError(f"FeatVolume: n_views must be positive, got {n_views}")
        self.feat_dim, self.view_embed_dim, self.feat_vol_reso = feat_dim, view_embed_dim, feat_vol_reso
        self.dir_norm = ModLN(feat_dim, SH_FEATURES, eps=1e-6)
        if view_embed_dim > 0:
            self.view_embed = nn.Parameter(torch.randn(1, n_views, view_embed_dim, 1, 1, 1) *
                                           (1. / view_embed_dim) ** 0.5)
        self.register_buffer("volume_grid", dense_grid(feat_vol_reso, scene_size))

    def forward(self, img_feats, rays_down, w2cs, ixts, image_hw) -> torch.Tensor:
        """``build_feat_vol``: [B,V,C,R,R,R]."""
        return self._run("FeatVolume.forward", img_feats, rays_down, w2cs, ixts, image_hw, 0)

    def cond_tokens(self, img_feats, rays_down, w2cs, ixts, image_hw, n_group: int) -> torch.Tensor:
        """``build_feat_vol``, the ``view_embed`` concatenation and ``VolTransformer.forward``'s blocks for
        ``n_group`` groups per axis: [B g^3, V bs^3, C+E] with bs = R / n_group."""
        fn = "FeatVolume.cond_tokens"
        R = self.feat_vol_reso
        if isinstance(n_group, bool) or not isinstance(n_group, int) or n_group < 1 or R % n_group != 0:
            raise RuntimeError(f"{fn}: n_group must be a positive divisor of {R}, got {n_group!r}")
        return self._run(fn, img_feats, rays_down, w2cs, ixts, image_hw, n_group)

    def _run(self, fn, img_feats, rays_down, w2cs, ixts, image_hw, n_group):
        C = self.feat_dim
        named = (("img_feats", img_feats), ("rays_down", rays_down), ("w2cs", w2cs), ("ixts", ixts))
        for name, t in named:
            if not isinstance(t, torch.Tensor):
                raise TypeError(f"{fn}: {name} must be a tensor")
        if rays_down.ndim != 5 or rays_down.shape[4] != 6:
            raise RuntimeError(f"{fn}: rays_down must be [B,V,h,w,6], got {tuple(rays_down.shape)}")
        B, V, h, w = (int(s) for s in rays_down.shape[:4])
        if B < 1 or not 1 <= V <= 8 or h < 1 or w < 1:
            raise RuntimeError(f"{fn}: rays_down must have B >= 1, 1 <= V <= 8 and h, w >= 1, "
                               f"got {tuple(rays_down.shape)}")
        for name, t, shape in (("img_feats", img_feats, (B * V, C, h, w)), ("w2cs", w2cs, (B, V, 4, 4)),
                               ("ixts", ixts, (B, V, 3, 3))):
            if tuple(t.shape) != shape:
                raise RuntimeError(f"{fn}: {name} must be {shape}, got {tuple(t.shape)}")
        if len(image_hw) != 2 or any(int(s) < 1 for s in image_hw):
            raise RuntimeError(f"{fn}: image_hw must be (H, W) with H, W >= 1, got {tuple(image_hw)}")
        E = self.view_embed_dim if n_group > 0 else 0
        ve = self.view_embed.view(self.view_embed.shape[1], E) if E > 0 else None
        if ve is not None and V > ve.shape[0]:
            raise RuntimeError(f"{fn}: {V} views but view_embed has {ve.shape[0]} rows")
        for name, t in named[1:]:
            if t.requires_grad:
                raise RuntimeError(f"{fn}: {name} requires grad, but the op treats it as a constant (as LaRa does); "
                                   "detach it")
        params = (self.dir_norm.norm.weight, self.dir_norm.norm.bias, self.dir_norm.mlp[1].weight,
                  self.dir_norm.mlp[1].bias)
        R = self.feat_vol_reso
        checked = [("dir_norm.norm.weight", params[0], (C,)), ("dir_norm.norm.bias", params[1], (C,)),
                   ("dir_norm.mlp.1.weight", params[2], (2 * C, SH_FEATURES)),
                   ("dir_norm.mlp.1.bias", params[3], (2 * C,)),
                   ("volume_grid", self.volume_grid, (R, R, R, 3))]
        if ve is not None:
            checked.append(("view_embed", ve, tuple(ve.shape)))
        for name, t, shape in checked:
            if tuple(t.shape) != shape:
                raise RuntimeError(f"{fn}: {name} must be {shape}, got {tuple(t.shape)}")
        autocast = torch.is_autocast_enabled("cuda")
        dev = img_feats.device
        for name, t in named:
            if not t.is_floating_point() or (not autocast and t.dtype != torch.float32):
                raise RuntimeError(f"{fn}: expected scalar type Float but found {t.dtype} for {name}")
            if not t.is_cuda or t.device != dev:
                raise RuntimeError(f"{fn}: {name} must be a CUDA tensor on {dev}, got {t.device}")
        for name, t, _ in checked:
            if t.dtype != torch.float32:
                raise RuntimeError(f"{fn}: expected scalar type Float but found {t.dtype} for {name}")
            if t.device != dev:
                raise RuntimeError(f"{fn}: {name} is on {t.device}, the inputs on {dev}")
        return _FeatVolume.apply(img_feats, rays_down, w2cs, ixts, self.volume_grid, ve,
                                 (int(image_hw[0]), int(image_hw[1])), n_group, *params)
