"""Views into the forward's workspaces (for tests and tooling).

The reference's opaque blobs can be parsed with the layout in
``rasterizer_impl.cu:155-194``; this is the equivalent for this package's layout, driven by
``srf_state_layout`` so the offsets never go stale.
"""
from __future__ import annotations

from typing import Dict

import torch

from . import _lib
from .rasterizer import ForwardState


class _View:
    """One view's slice of a batched ForwardState (V back-to-back workspaces)."""

    def __init__(self, state: ForwardState, view: int):
        V = state.nviews
        def cut(t):
            n = t.numel() // V
            return t[view * n:(view + 1) * n]
        self.geom, self.tile, self.image, self.point_list = cut(state.geom), cut(state.tile), cut(state.image), cut(state.point_list)
        self.num_rendered = state.resolve()[view]


def unpack_state(state: ForwardState, P: int, H: int, W: int, view: int = 0) -> Dict[str, torch.Tensor]:
    if state.nviews > 1:
        state = _View(state, view)
    lib = _lib.load()
    g_off, t_off, i_off = _lib.layout(lib, P, H, W)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    ntiles = gx * gy
    npix = H * W
    R = state.num_rendered
    out: Dict[str, torch.Tensor] = {}
    if P > 0:
        rec = state.geom[g_off[0]:g_off[0] + 96 * P].view(torch.float32).view(P, 24)
        out["rec"] = rec
        out["transMat"] = rec[:, [0, 2, 4, 1, 3, 5, 6, 7, 8]]     # record interleaves Tu / Tv (surfel_common.cuh)
        out["means2D"] = rec[:, 9:11]
        out["opacity"] = rec[:, 11]
        out["normal"] = rec[:, 12:15]
        out["depths_rec"] = rec[:, 15]
        out["rgb"] = rec[:, 16:19]
        out["clamp_bits"] = rec[:, 19].view(torch.int32)
        out["depths"] = state.geom[g_off[1]:g_off[1] + 4 * P].view(torch.float32)
        rects = state.geom[g_off[2]:g_off[2] + 8 * P].view(torch.int32).view(P, 2)
        out["rect"] = torch.stack([rects[:, 0] & 0xFFFF, (rects[:, 0] >> 16) & 0xFFFF,
                                   rects[:, 1] & 0xFFFF, (rects[:, 1] >> 16) & 0xFFFF], dim=1)
        out["tiles_touched"] = (out["rect"][:, 2] - out["rect"][:, 0]) * (out["rect"][:, 3] - out["rect"][:, 1])
    out["tile_count"] = state.tile[t_off[0]:t_off[0] + 256 * ntiles].view(torch.int32).view(ntiles, 64)[:, 0]
    out["counters"] = state.tile[t_off[1]:t_off[1] + 16].view(torch.int32)
    out["ranges"] = state.tile[t_off[2]:t_off[2] + 8 * ntiles].view(torch.int32).view(ntiles, 2)
    out["accum"] = state.image[i_off[0]:i_off[0] + 12 * npix].view(torch.float32).view(3, H, W)
    out["n_contrib"] = state.image[i_off[1]:i_off[1] + 8 * npix].view(torch.int32).view(2, H, W)
    out["point_list"] = state.point_list[:4 * R].view(torch.int32) if R > 0 else state.point_list[:0].view(torch.int32)
    return out
