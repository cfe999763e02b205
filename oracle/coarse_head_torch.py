"""Plain-torch restatement of LaRa's coarse-pass decoder head (``Decoder.forward_coarse``, lightning/network.py:259-278:
``mlp_coarse`` and the split of its output, optionally followed by ``Network.get_offseted_pt``, :425-429), the checker
of lara_b200/csrc/coarse_head.cu.  On the CPU it reproduces LaRa's values and gradients bit for bit
(tests/test_coarse_head.py); in float64 it is the accuracy reference of the kernels.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.torch_restatements import decoder_layout_torch


def mlp_coarse_torch(feats, params):
    """Linear, ReLU, Linear, ReLU, Linear with params (w0, b0, w1, b1, w2, b2)."""
    w0, b0, w1, b1, w2, b2 = params
    return F.linear(F.relu(F.linear(F.relu(F.linear(feats, w0, b0)), w1, b1)), w2, b2)


def coarse_head_torch(feats, params, K, sh_dim, opacity_shift, scaling_shift, group_centers=None, half_cell_size=None):
    """feats [B, ..., D] -> (offset or centers, sh, scaling, rotation, opacity) as LaRa computes them: the offset form
    without group_centers, else the centers form."""
    parameters = mlp_coarse_torch(feats, params).float()
    if group_centers is not None:
        B = parameters.shape[0]
        return decoder_layout_torch(parameters.reshape(B, -1, parameters.shape[-1]), group_centers, K, sh_dim,
                                    opacity_shift, scaling_shift, half_cell_size)
    parameters = parameters.view(*parameters.shape[:-1], K, -1)
    offset, sh, opacity, scaling, rotation = torch.split(parameters, [3, sh_dim, 1, 2, 4], dim=-1)
    opacity = opacity + opacity_shift
    scaling = scaling + scaling_shift
    offset = torch.sigmoid(offset) * 2 - 1.0
    B = opacity.shape[0]
    return (offset.view(B, -1, 3), sh.view(B, -1, sh_dim // 3, 3), scaling.view(B, -1, 2), rotation.view(B, -1, 4),
            opacity.view(B, -1, 1))
