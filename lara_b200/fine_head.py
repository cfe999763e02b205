"""Fused fine-pass decoder head of LaRa (``Decoder.forward_fine``, lightning/network.py:280-284, with the mask gathers
and residual of :508-512) -- an additional entry point next to the unchanged rasterizer.

``FineHead`` holds the fine part of LaRa's ``Decoder`` under LaRa's own parameter names (``norm``, ``cross_att``,
``mlp_fine``), so ``FineHead(D, sh_dim).load_state_dict(decoder.state_dict(), strict=False)`` picks it up.  Its two
entries run on one CUDA kernel per direction (include/surfel_fine_head.h):

* ``forward_fine(volume_feat [n,D], point_feats [n,V,8]) -> [n,1,sh_dim]`` is the drop-in for
  ``Decoder.forward_fine``;
* ``fine_shs(volume_feat_up [N,D], K, mask [N*K], point_feats [V,8,n], shs_coarse [N*K,M,3]) -> [n,M,3]`` replaces
  network.py:508-512 in one call: the voxel-row gather, the einsum of the point features, the head and the residual.
  ``point_feats`` is what ``sample_point_feats`` returns.

The backward recomputes the head per tile of points, so autograd keeps only the inputs, and it is bit-reproducible
with or without ``torch.use_deterministic_algorithms`` (no atomics; DESIGN §3.16).  Differences from the reference, by
design: the head always computes in fp32 -- under bf16 autocast LaRa's linears and attention would run in bf16 -- and
its fp32 rounding differs from torch's (the head algebra is reassociated), within 1e-5 of each tensor's maximum.
"""
from __future__ import annotations

import torch
from torch import nn

from . import _lib

HEADS, COND, HIDDEN = 8, 8, 64
SH_DIMS = (3, 12, 27, 48)
_PARAMS = ("norm.weight", "norm.bias", "cross_att.q_proj_weight", "cross_att.k_proj_weight",
           "cross_att.v_proj_weight", "cross_att.out_proj.weight", "mlp_fine.0.weight", "mlp_fine.0.bias",
           "mlp_fine.2.weight", "mlp_fine.2.bias")


def _check_tensors(fn, named):
    """dtype / device / contiguity checks before any launch: the kernels take raw pointers."""
    dev = named[0][1].device
    for name, t in named:
        if t.dtype != torch.float32:
            raise RuntimeError(f"{fn}: expected scalar type Float but found {t.dtype} for {name}")
        if not t.is_cuda or t.device != dev:
            raise RuntimeError(f"{fn}: {name} must be a CUDA tensor on {dev}, got {t.device}")
        if not t.is_contiguous():
            raise RuntimeError(f"{fn}: {name} must be contiguous")


class _FineHead(torch.autograd.Function):
    """(volume_feat, point_feats [V,8,n], shs_coarse or None, idx or None, K, *params) -> sh [n, sh_dim]."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, vf, pf, shs, idx, K, *params):
        vf, pf = vf.contiguous(), pf.contiguous()
        shs = shs.contiguous() if shs is not None else None
        V, _, n = (int(s) for s in pf.shape)
        D, S = int(vf.shape[1]), int(params[8].shape[0])
        N = int(vf.shape[0])
        out = torch.empty((n, S), dtype=torch.float32, device=vf.device)
        _lib.launch("srf_fine_head_forward", vf.device, n, V, D, S, K, N, vf.data_ptr(),
                    idx.data_ptr() if idx is not None else None, pf.data_ptr(),
                    shs.data_ptr() if shs is not None else None, *[p.data_ptr() for p in params], out.data_ptr())
        ctx.save_for_backward(vf, pf, idx, *params)
        ctx.dims = (n, V, D, S, K, N, shs is not None, None if shs is None else shs.shape)
        return out

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, g):
        vf, pf, idx, *params = ctx.saved_tensors
        n, V, D, S, K, N, has_shs, shs_shape = ctx.dims
        dev = vf.device
        g = g.contiguous()
        g_vf, g_pf = torch.empty_like(vf), torch.empty_like(pf)
        g_shs = torch.empty(shs_shape, dtype=torch.float32, device=dev) if has_shs else None
        g_params = [torch.empty_like(p) for p in params]
        gather = idx is not None
        with _lib._DeviceGuard(dev):        # the workspace size depends on the device's SM count
            ws = torch.empty(_lib.fine_head_workspace_bytes(_lib.load(), n, V, D, S, gather), dtype=torch.uint8,
                             device=dev)
        _lib.launch("srf_fine_head_backward", dev, n, V, D, S, K, N, vf.data_ptr(), idx.data_ptr() if gather else None,
                    pf.data_ptr(), *[p.data_ptr() for p in params], g.data_ptr(), ws.data_ptr(), g_vf.data_ptr(),
                    g_pf.data_ptr(), g_shs.data_ptr() if has_shs else None, *[p.data_ptr() for p in g_params])
        return (g_vf, g_pf, g_shs, None, None, *g_params)


class FineHead(nn.Module):
    """The fine part of LaRa's ``Decoder`` (network.py:233-240): ``norm``, ``cross_att`` and ``mlp_fine``, with
    LaRa's names, shapes and initialisation.  ``cross_att`` is a ``nn.MultiheadAttention`` used only as the holder of
    the four projection weights; the computation is the fused kernel's."""

    def __init__(self, in_dim: int = 80, sh_dim: int = 12):
        super().__init__()
        if in_dim % 8 != 0 or not 8 <= in_dim <= 128:
            raise ValueError(f"FineHead: in_dim must be a multiple of 8 up to 128, got {in_dim}")
        if sh_dim not in SH_DIMS:
            raise ValueError(f"FineHead: sh_dim must be one of {SH_DIMS}, got {sh_dim}")
        self.in_dim, self.sh_dim = in_dim, sh_dim
        self.norm = nn.LayerNorm(in_dim)
        self.cross_att = nn.MultiheadAttention(embed_dim=in_dim, num_heads=HEADS, kdim=COND, vdim=COND, dropout=0.0,
                                               bias=False, batch_first=True)
        self.mlp_fine = nn.Sequential(nn.Linear(in_dim, HIDDEN), nn.ReLU(), nn.Linear(HIDDEN, sh_dim))
        for layer in self.mlp_fine:                # Decoder.init: xavier weights, zero biases
            if isinstance(layer, nn.Linear):
                nn.init.xavier_uniform_(layer.weight.data)
                nn.init.zeros_(layer.bias.data)

    def _params(self):
        """The ten tensors in the kernel's order.  At in_dim 8 (= kdim) nn.MultiheadAttention, as in LaRa, keeps the
        three projections packed in ``in_proj_weight``; its row blocks are used then."""
        a = self.cross_att
        if a._qkv_same_embed_dim:
            wq, wk, wv = a.in_proj_weight.chunk(3)
        else:
            wq, wk, wv = a.q_proj_weight, a.k_proj_weight, a.v_proj_weight
        return (self.norm.weight, self.norm.bias, wq, wk, wv, a.out_proj.weight, self.mlp_fine[0].weight,
                self.mlp_fine[0].bias, self.mlp_fine[2].weight, self.mlp_fine[2].bias)

    def _checked_params(self, fn):
        params = self._params()
        _check_tensors(fn, list(zip(_PARAMS, params)))
        return params

    def forward_fine(self, volume_feat: torch.Tensor, point_feats: torch.Tensor) -> torch.Tensor:
        """``Decoder.forward_fine``: volume_feat [n,D], point_feats [n,V,8] -> sh [n,1,sh_dim]."""
        fn = "FineHead.forward_fine"
        D = self.in_dim
        if volume_feat.ndim != 2 or volume_feat.shape[1] != D:
            raise RuntimeError(f"{fn}: volume_feat must be [n,{D}], got {tuple(volume_feat.shape)}")
        n = int(volume_feat.shape[0])
        if point_feats.ndim != 3 or point_feats.shape[0] != n or point_feats.shape[2] != COND \
                or not 1 <= point_feats.shape[1] <= 8:
            raise RuntimeError(f"{fn}: point_feats must be [{n},V,8] with 1 <= V <= 8, got {tuple(point_feats.shape)}")
        params = self._prepared(fn, volume_feat, point_feats)
        pf = point_feats.permute(1, 2, 0).contiguous()      # the kernel reads [V,8,n]
        return _FineHead.apply(volume_feat, pf, None, None, 1, *params).unsqueeze(1)

    def fine_shs(self, volume_feat_up: torch.Tensor, K: int, mask, point_feats: torch.Tensor,
                 shs_coarse: torch.Tensor) -> torch.Tensor:
        """network.py:508-512 in one call: ``_shs_fine`` [n,M,3] of the masked Gaussians.

        One scene: volume_feat_up [N,D] (its voxel features), K Gaussians per voxel, mask [N*K] bool (after
        ``_check_mask``), point_feats [V,8,n] (``sample_point_feats``' output for those n Gaussians), shs_coarse
        [N*K,M,3] with 3 M = sh_dim.

        All B scenes of a batch in one call: volume_feat_up [B,N,D], ``mask`` the
        :class:`lara_b200.multiview.FineSubset` of the masks [B,N*K] (or those masks), point_feats [V,8,n]
        (``sample_batch_point_feats``' output) and shs_coarse [B,N*K,M,3]; returns [n,M,3] in scene order, what
        ``render_batch_subset_views`` takes.  Each row is bit for bit the one-scene call's; the parameter gradients are
        summed over all scenes at once."""
        fn = "FineHead.fine_shs"
        D, S = self.in_dim, self.sh_dim
        if isinstance(K, bool) or not isinstance(K, int) or K < 1:
            raise RuntimeError(f"{fn}: K must be a positive int, got {K!r}")
        if volume_feat_up.ndim == 3:
            return self._fine_shs_batch(fn, volume_feat_up, K, mask, point_feats, shs_coarse)
        if volume_feat_up.ndim != 2 or volume_feat_up.shape[1] != D:
            raise RuntimeError(f"{fn}: volume_feat_up must be [N,{D}], got {tuple(volume_feat_up.shape)}")
        NK = int(volume_feat_up.shape[0]) * K
        if mask.dtype != torch.bool or tuple(mask.shape) != (NK,):
            raise RuntimeError(f"{fn}: mask must be a bool tensor of shape ({NK},), got {mask.dtype} "
                               f"{tuple(mask.shape)}")
        if tuple(shs_coarse.shape) != (NK, S // 3, 3):
            raise RuntimeError(f"{fn}: shs_coarse must be {(NK, S // 3, 3)}, got {tuple(shs_coarse.shape)}")
        self._check_point_feats(fn, point_feats)
        if NK >= 2 ** 31:
            raise RuntimeError(f"{fn}: N*K = {NK} is over the int32 index range")
        params = self._prepared(fn, volume_feat_up, point_feats, shs_coarse)
        if not mask.is_cuda or mask.device != volume_feat_up.device:
            raise RuntimeError(f"{fn}: mask must be a CUDA tensor on {volume_feat_up.device}, got {mask.device}")
        idx = mask.nonzero().squeeze(1).to(torch.int32)          # strictly increasing by construction
        n = int(idx.shape[0])
        if point_feats.shape[2] != n:
            raise RuntimeError(f"{fn}: point_feats has {point_feats.shape[2]} points but mask selects {n}")
        out = _FineHead.apply(volume_feat_up, point_feats, shs_coarse.reshape(NK, S), idx, K, *params)
        return out.view(n, S // 3, 3)

    @staticmethod
    def _check_point_feats(fn, point_feats):
        if not isinstance(point_feats, torch.Tensor) or point_feats.ndim != 3 or point_feats.shape[1] != COND or \
                not 1 <= point_feats.shape[0] <= 8:
            raise RuntimeError(f"{fn}: point_feats must be [V,8,n] with 1 <= V <= 8, got "
                               f"{tuple(getattr(point_feats, 'shape', ()))}")

    def _fine_shs_batch(self, fn, volume_feat_up, K, subset, point_feats, shs_coarse):
        """The batch form of :meth:`fine_shs`: the subset's global rows b*N*K + i index the flattened [B*N*K] Gaussians,
        so the kernel's voxel row, row // K, is b*N + i // K of the flattened [B*N, D] features."""
        from .multiview import FineSubset
        D, S = self.in_dim, self.sh_dim
        if volume_feat_up.shape[2] != D:
            raise RuntimeError(f"{fn}: volume_feat_up must be [B,N,{D}], got {tuple(volume_feat_up.shape)}")
        B, N = int(volume_feat_up.shape[0]), int(volume_feat_up.shape[1])
        NK = N * K
        if isinstance(subset, torch.Tensor):
            if subset.dtype != torch.bool or tuple(subset.shape) != (B, NK):
                raise RuntimeError(f"{fn}: masks must be a bool tensor of shape ({B}, {NK}), got {subset.dtype} "
                                   f"{tuple(subset.shape)}")
            if B * NK >= 2 ** 31:
                raise RuntimeError(f"{fn}: B*N*K = {B * NK} is over the int32 index range")
            if not subset.is_cuda or subset.device != volume_feat_up.device:
                raise RuntimeError(f"{fn}: masks must be a CUDA tensor on {volume_feat_up.device}, got {subset.device}")
            subset = FineSubset(subset)
        elif not isinstance(subset, FineSubset):
            raise RuntimeError(f"{fn}: with volume_feat_up [B,N,D], mask must be a FineSubset or bool masks [B,N*K], "
                               f"got {type(subset).__name__}")
        if (subset.scenes, subset.P) != (B, NK):
            raise RuntimeError(f"{fn}: the subset's masks are [{subset.scenes},{subset.P}], expected [{B},{NK}]")
        if B * NK >= 2 ** 31:
            raise RuntimeError(f"{fn}: B*N*K = {B * NK} is over the int32 index range")
        if tuple(shs_coarse.shape) != (B, NK, S // 3, 3):
            raise RuntimeError(f"{fn}: shs_coarse must be {(B, NK, S // 3, 3)}, got {tuple(shs_coarse.shape)}")
        self._check_point_feats(fn, point_feats)
        params = self._prepared(fn, volume_feat_up, point_feats, shs_coarse)
        if subset.rows.device != volume_feat_up.device:
            raise RuntimeError(f"{fn}: the subset is on {subset.rows.device}, volume_feat_up on {volume_feat_up.device}")
        n = subset.n
        if point_feats.shape[2] != n:
            raise RuntimeError(f"{fn}: point_feats has {point_feats.shape[2]} points but the masks select {n}")
        if n == 0:          # nothing selected: no launch, an empty result that still leads back to shs_coarse
            return shs_coarse.reshape(B * NK, S // 3, 3)[:0]
        out = _FineHead.apply(volume_feat_up.reshape(B * N, D), point_feats, shs_coarse.reshape(B * NK, S),
                              subset.rows, K, *params)
        return out.view(n, S // 3, 3)

    def _prepared(self, fn, *inputs):
        """Argument checks of the inputs (fp32 or, under autocast, any float type) and the parameters."""
        dtype = torch.float32 if torch.is_autocast_enabled("cuda") else None
        names = ("volume_feat", "point_feats", "shs_coarse")
        for name, t in zip(names, inputs):
            if not isinstance(t, torch.Tensor):
                raise TypeError(f"{fn}: {name} must be a tensor")
            if dtype is None and t.dtype != torch.float32:
                raise RuntimeError(f"{fn}: expected scalar type Float but found {t.dtype} for {name}")
            if not t.is_floating_point():
                raise RuntimeError(f"{fn}: expected a floating-point {name}, got {t.dtype}")
        dev = inputs[0].device
        for name, t in zip(names, inputs):
            if not t.is_cuda or t.device != dev:
                raise RuntimeError(f"{fn}: {name} must be a CUDA tensor on {dev}, got {t.device}")
        params = self._checked_params(fn)
        if params[0].device != dev:
            raise RuntimeError(f"{fn}: the parameters are on {params[0].device}, the inputs on {dev}")
        return params
