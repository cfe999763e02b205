"""Decoder epilogue (SURVEY.md 8f rank 4) -- an additional entry point.

``Decoder.forward_coarse`` (``lightning/network.py:259-278``) turns the MLP output ``[B, N, K*C]`` into five tensors
with a ``view`` + ``torch.split`` -- strided views, so ``sh`` and ``rotation`` are re-packed by ``.contiguous()`` inside
every one of the 8-16 rasterizer calls of a scene -- plus two shift kernels and ``sigmoid(offset)*2-1``;
``Network.get_offseted_pt`` (``:425-429``) then adds the voxel centres.  ``gaussians_from_decoder`` does all of it
in one CUDA pass and hands back the five CONTIGUOUS tensors the rasterizer's preprocess kernel loads with vector
instructions (and one mirror-image pass in the backward).  A maintainer switches ``forward_coarse`` to it with::

    parameters = self.mlp_coarse(feats).float()
    return gaussians_from_decoder(parameters, group_centers, self.K, self.sh_dim, opacity_shift, scaling_shift, half_cell)
"""
from __future__ import annotations

from typing import Tuple

import torch

from . import _lib
from ._lib import _contig, _ptr


class _DecoderLayout(torch.autograd.Function):
    @staticmethod
    def forward(ctx, params, group_centers, K, sh_dim, opacity_shift, scaling_shift, half_cell):
        if params.ndim != 3:
            raise RuntimeError("gaussians_from_decoder: parameters must be [B, N, K*C]")
        B, N, KC = params.shape
        C = 10 + int(sh_dim)
        if KC != int(K) * C or sh_dim % 3 != 0:
            raise RuntimeError(f"gaussians_from_decoder: last dim {KC} != K*(10+sh_dim) = {int(K) * C}")
        gc = group_centers.reshape(-1, 3)
        if gc.shape[0] != N:
            raise RuntimeError(f"gaussians_from_decoder: group_centers must hold N = {N} voxel centres, got {gc.shape[0]}")
        for name, t in (("parameters", params), ("group_centers", gc)):
            if not t.is_cuda or t.dtype != torch.float32 or t.device != params.device:
                raise RuntimeError(f"gaussians_from_decoder: {name} must be a float32 CUDA tensor on {params.device}")
        params_c, gc = params.contiguous(), gc.contiguous()
        dev = params.device
        G = N * int(K)

        def new(*shape):
            return torch.empty(shape, dtype=torch.float32, device=dev)
        centers, shs, opacity = new(B, G, 3), new(B, G, sh_dim // 3, 3), new(B, G, 1)
        scaling, rotation = new(B, G, 2), new(B, G, 4)
        _lib.launch("srf_decoder_layout_forward", dev, B, N, int(K), int(sh_dim), float(opacity_shift),
                    float(scaling_shift), float(half_cell), params_c.data_ptr(), gc.data_ptr(), centers.data_ptr(),
                    shs.data_ptr(), opacity.data_ptr(), scaling.data_ptr(), rotation.data_ptr())
        ctx.save_for_backward(params_c)
        ctx.meta = (B, N, int(K), int(sh_dim), float(half_cell))
        return centers, shs, scaling, rotation, opacity

    @staticmethod
    def backward(ctx, g_centers, g_shs, g_scaling, g_rotation, g_opacity):
        (params,) = ctx.saved_tensors
        B, N, K, sh_dim, half_cell = ctx.meta
        g_centers, g_shs, g_scaling, g_rotation, g_opacity = map(
            _contig, (g_centers, g_shs, g_scaling, g_rotation, g_opacity))
        g_params = torch.empty_like(params)
        _lib.launch("srf_decoder_layout_backward", params.device, B, N, K, sh_dim, half_cell, params.data_ptr(),
                    _ptr(g_centers), _ptr(g_shs), _ptr(g_opacity), _ptr(g_scaling), _ptr(g_rotation),
                    g_params.data_ptr())
        return g_params, None, None, None, None, None, None


def gaussians_from_decoder(parameters: torch.Tensor, group_centers: torch.Tensor, K: int, sh_dim: int,
                           opacity_shift: float, scaling_shift: float, half_cell_size: float
                           ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """(centers [B,N*K,3], shs [B,N*K,sh_dim/3,3], scaling [B,N*K,2], rotation [B,N*K,4], opacity [B,N*K,1]):
    the return order of ``Decoder.forward_coarse`` with ``offset`` already turned into ``centers`` by
    ``get_offseted_pt``; all contiguous.  ``parameters`` is the fp32 MLP output [B, N, K*(10+sh_dim)],
    ``group_centers`` [N,3] (or [1,N,3]), ``half_cell_size = 0.5*scene_size/n_offset_groups``."""
    return _DecoderLayout.apply(parameters, group_centers, int(K), int(sh_dim), float(opacity_shift), float(scaling_shift),
                                float(half_cell_size))
