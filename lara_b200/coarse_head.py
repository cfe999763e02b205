"""Fused coarse-pass decoder head of LaRa (``Decoder.forward_coarse``, lightning/network.py:259-278, optionally with
``Network.get_offseted_pt``, :425-429) -- an additional entry point next to the unchanged rasterizer.

``CoarseHead`` holds ``mlp_coarse`` under LaRa's own name and layout (``nn.Sequential`` of Linear(D,D), ReLU,
Linear(D,D), ReLU, Linear(D, K*(10+sh_dim))), so ``CoarseHead(D, sh_dim, K).load_state_dict(decoder.state_dict(),
strict=False)`` picks it up.  Its two entries run the three layers and the decoder layout in one CUDA kernel per
direction (include/surfel_coarse_head.h):

* ``forward_coarse(feats [B,...,D], opacity_shift, scaling_shift) -> (offset, sh, scaling, rotation, opacity)`` is the
  drop-in for ``Decoder.forward_coarse``;
* ``gaussians(feats, group_centers, opacity_shift, scaling_shift, half_cell_size) -> (centers, shs, scaling, rotation,
  opacity)`` adds ``get_offseted_pt``: what ``gaussians_from_decoder`` returns, ready for
  ``render_scene_views(..., raw_activations=True)``.

Autograd keeps only ``feats`` and the weights: the backward recomputes the MLP per tile of rows.  It is
bit-reproducible with or without ``torch.use_deterministic_algorithms`` (no atomics; DESIGN §3.20).  Differences from
LaRa, by design: the outputs are contiguous (LaRa returns strided views of the MLP output); they are fp32 under bf16
autocast, where LaRa's linears run in bf16; and the products are 3xTF32 tensor-core MMAs with fp32 accumulation, whose
rounding differs from cuBLAS's fp32 GEMMs (within 1e-5 of each tensor's maximum).
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
from torch import nn

from . import _lib

SH_DIMS = (3, 12, 27, 48)
_PARAMS = ("mlp_coarse.0.weight", "mlp_coarse.0.bias", "mlp_coarse.2.weight", "mlp_coarse.2.bias",
           "mlp_coarse.4.weight", "mlp_coarse.4.bias")


class _CoarseHead(torch.autograd.Function):
    """(feats [rows,D], group_centers [N,3] or None, N, K, sh_dim, opacity_shift, scaling_shift, half_cell, *params)
    -> the five [rows*K, ...] outputs of the layout."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, feats, gc, N, K, S, opacity_shift, scaling_shift, half_cell, *params):
        feats = feats.contiguous()
        rows, D = (int(s) for s in feats.shape)
        G, dev = rows * K, feats.device

        def new(*shape):
            return torch.empty(shape, dtype=torch.float32, device=dev)
        first, shs, opacity, scaling, rotation = new(G, 3), new(G, S), new(G), new(G, 2), new(G, 4)
        _lib.launch("srf_coarse_head_forward", dev, rows, N, D, K, S, opacity_shift, scaling_shift, half_cell,
                    feats.data_ptr(), _lib._ptr(gc), *[p.data_ptr() for p in params], first.data_ptr(),
                    shs.data_ptr(), opacity.data_ptr(), scaling.data_ptr(), rotation.data_ptr())
        ctx.save_for_backward(feats, gc, *params)
        ctx.dims = (rows, N, D, K, S, half_cell)
        return first, shs, scaling, rotation, opacity

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, g_first, g_shs, g_scaling, g_rotation, g_opacity):
        feats, gc, *params = ctx.saved_tensors
        rows, N, D, K, S, half_cell = ctx.dims
        dev = feats.device
        g_first, g_shs, g_scaling, g_rotation, g_opacity = map(
            _lib._contig, (g_first, g_shs, g_scaling, g_rotation, g_opacity))
        g_feats = torch.empty_like(feats)
        g_params = [torch.empty_like(p) for p in params]
        with _lib._DeviceGuard(dev):        # the workspace size depends on the device's SM count
            ws = torch.empty(_lib.coarse_head_workspace_bytes(_lib.load(), rows, D, K, S), dtype=torch.uint8,
                             device=dev)
        _lib.launch("srf_coarse_head_backward", dev, rows, N, D, K, S, half_cell, feats.data_ptr(), _lib._ptr(gc),
                    *[p.data_ptr() for p in params], _lib._ptr(g_first), _lib._ptr(g_shs), _lib._ptr(g_opacity),
                    _lib._ptr(g_scaling), _lib._ptr(g_rotation), ws.data_ptr(), g_feats.data_ptr(),
                    *[p.data_ptr() for p in g_params])
        return (g_feats, None, None, None, None, None, None, None, *g_params)


class CoarseHead(nn.Module):
    """The coarse part of LaRa's ``Decoder`` (network.py:226-230): ``mlp_coarse`` with LaRa's names, shapes and
    initialisation (xavier-uniform weights, zero biases)."""

    def __init__(self, in_dim: int = 80, sh_dim: int = 12, K: int = 2):
        super().__init__()
        if in_dim % 16 != 0 or not 16 <= in_dim <= 128:
            raise ValueError(f"CoarseHead: in_dim must be a multiple of 16 in [16, 128], got {in_dim}")
        if sh_dim not in SH_DIMS:
            raise ValueError(f"CoarseHead: sh_dim must be one of {SH_DIMS}, got {sh_dim}")
        if isinstance(K, bool) or not isinstance(K, int) or not 1 <= K <= 4:
            raise ValueError(f"CoarseHead: K must be an int in [1, 4], got {K!r}")
        self.in_dim, self.sh_dim, self.K = in_dim, sh_dim, K
        out_dim = K * (10 + sh_dim)
        self.mlp_coarse = nn.Sequential(nn.Linear(in_dim, in_dim), nn.ReLU(), nn.Linear(in_dim, in_dim), nn.ReLU(),
                                        nn.Linear(in_dim, out_dim))
        for layer in self.mlp_coarse:              # Decoder.init: xavier weights, zero biases
            if isinstance(layer, nn.Linear):
                nn.init.xavier_uniform_(layer.weight.data)
                nn.init.zeros_(layer.bias.data)

    def _params(self):
        m = self.mlp_coarse
        return (m[0].weight, m[0].bias, m[2].weight, m[2].bias, m[4].weight, m[4].bias)

    def _run(self, fn, feats, group_centers, opacity_shift, scaling_shift, half_cell):
        D, K, S = self.in_dim, self.K, self.sh_dim
        if not isinstance(feats, torch.Tensor):
            raise TypeError(f"{fn}: feats must be a tensor")
        if feats.ndim < 2 or feats.shape[-1] != D:
            raise RuntimeError(f"{fn}: feats must be [B, ..., {D}], got {tuple(feats.shape)}")
        if not feats.is_floating_point():
            raise RuntimeError(f"{fn}: expected a floating-point feats, got {feats.dtype}")
        if not torch.is_autocast_enabled("cuda") and feats.dtype != torch.float32:
            raise RuntimeError(f"{fn}: expected scalar type Float but found {feats.dtype} for feats")
        dev = feats.device
        if not feats.is_cuda:
            raise RuntimeError(f"{fn}: feats must be a CUDA tensor, got {dev}")
        B = int(feats.shape[0])
        rows = feats.numel() // D
        N = rows // B if B > 0 else 0
        if rows * K >= 2 ** 31:
            raise RuntimeError(f"{fn}: rows*K = {rows * K} is over the int32 index range")
        gc = None
        if group_centers is not None:
            gc = group_centers.reshape(-1, 3)
            if gc.shape[0] != N:
                raise RuntimeError(f"{fn}: group_centers must hold N = {N} voxel centres, got {gc.shape[0]}")
            if gc.dtype != torch.float32 or not gc.is_cuda or gc.device != dev:
                raise RuntimeError(f"{fn}: group_centers must be a float32 CUDA tensor on {dev}")
            gc = gc.contiguous()
        params = self._params()
        for name, p in zip(_PARAMS, params):
            if p.dtype != torch.float32:
                raise RuntimeError(f"{fn}: expected scalar type Float but found {p.dtype} for {name}")
            if not p.is_cuda or p.device != dev:
                raise RuntimeError(f"{fn}: {name} is on {p.device}, feats on {dev}")
        x = feats.reshape(rows, D)
        outs = _CoarseHead.apply(x, gc, max(N, 1), K, S, float(opacity_shift), float(scaling_shift),
                                 float(half_cell), *params)
        first, shs, scaling, rotation, opacity = outs
        G = N * K
        return (first.view(B, G, 3), shs.view(B, G, S // 3, 3), scaling.view(B, G, 2), rotation.view(B, G, 4),
                opacity.view(B, G, 1))

    def forward_coarse(self, feats: torch.Tensor, opacity_shift: float, scaling_shift: float
                       ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
        """``Decoder.forward_coarse``: feats [B, ..., D] -> (offset [B,N*K,3], sh [B,N*K,sh_dim/3,3], scaling
        [B,N*K,2], rotation [B,N*K,4], opacity [B,N*K,1]) with N the voxels per scene; all contiguous fp32."""
        return self._run("CoarseHead.forward_coarse", feats, None, opacity_shift, scaling_shift, 1.0)

    def gaussians(self, feats: torch.Tensor, group_centers: Optional[torch.Tensor], opacity_shift: float,
                  scaling_shift: float, half_cell_size: float
                  ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
        """``forward_coarse`` + ``get_offseted_pt``: (centers, shs, scaling, rotation, opacity), what
        ``gaussians_from_decoder`` returns.  group_centers [N,3] (or [1,N,3]), ``half_cell_size =
        0.5*scene_size/n_offset_groups``."""
        if group_centers is None:
            raise RuntimeError("CoarseHead.gaussians: group_centers is required (forward_coarse returns offsets)")
        return self._run("CoarseHead.gaussians", feats, group_centers, opacity_shift, scaling_shift, half_cell_size)
