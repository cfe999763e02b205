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
        self.capacity = state.capacity


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
    # the blend forward's contribution record, after the list in the same workspace (include/surfel_rasterizer.h):
    # [8 warp blocks, R list positions], bit l = the splat was blended into pixel l of the tile's 8x4 block
    cap = state.capacity
    moff = (4 * cap + 255) // 256 * 256
    out["contrib_masks"] = state.point_list[moff:moff + 32 * cap].view(torch.int32).view(8, cap)[:, :R]
    return out


def unpack_ms_ssim(ws: torch.Tensor, B: int, C: int, H: int, W: int) -> Dict[str, object]:
    """Views into a fused MS-SSIM workspace (uint8, srf_ms_ssim_workspace_bytes) of the logical B x C x H x W image,
    through ``srf_ms_ssim_workspace_layout``: ``X``, ``Y``, ``dX`` lists over the levels of [B,C,h_l,w_l] tensors
    (None at level 0, which lives in the caller's tensors), ``part`` (list of [B*C, tiles] double), ``mean``
    [5,B,C] double, ``val`` [B,C] double, ``coef`` [5,B,C] float, and the geometry under ``layout``."""
    L = _lib.ms_ssim_layout(_lib.load(), B, C, H, W)
    P = B * C

    def f32(off, n):
        return ws[off:off + 4 * n].view(torch.float32)

    out: Dict[str, object] = {"layout": L, "X": [None], "Y": [None], "dX": [None], "part": []}
    for l in range(5):
        h, w = L["h"][l], L["w"][l]
        n = P * h * w
        if l:
            xy = f32(L["pyr"] + 4 * L["pyr_l"][l], 2 * n).view(2, B, C, h, w)
            out["X"].append(xy[0])
            out["Y"].append(xy[1])
            out["dX"].append(f32(L["gpyr"] + 4 * L["gpyr_l"][l], n).view(B, C, h, w))
        nt = L["ntx"][l] * L["nty"][l]
        off = L["part"] + 8 * L["part_l"][l]
        out["part"].append(ws[off:off + 8 * P * nt].view(torch.float64).view(P, nt))
    out["mean"] = ws[L["mean"]:L["mean"] + 8 * 5 * P].view(torch.float64).view(5, B, C)
    out["val"] = ws[L["val"]:L["val"] + 8 * P].view(torch.float64).view(B, C)
    out["coef"] = f32(L["coef"], 5 * P).view(5, B, C)
    return out
