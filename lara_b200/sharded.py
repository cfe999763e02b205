"""View-sharded rasterization: the multi-GPU form of the hot path (SURVEY.md 8e).

Every target view of a scene is an independent forward+backward over the same read-only
Gaussian set; only the parameter gradients sum across views.  One process per GPU
(``torch.distributed``, NCCL over NVLink): rank r renders views ``r, r+G, r+2G, ...`` in ONE
launch set (``srf_scenes_*`` with one scene), the per-Gaussian backward sums the rank's views in registers and adds
the result into one flat fp32 buffer (segment-major: means3D | sh | opacity | scales | rotations),
and a single ``all_reduce(sum)`` of that buffer finishes the step.  Images / aux maps stay on the rank
that owns the view.  The reference has nothing like this (it is single-GPU; LaRa only
data-parallelises over scenes), so there is no reference API to mirror here -- this is an
additional entry point next to the unchanged per-view one.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence, Tuple

import torch

from . import rasterizer as R


def shard_views(num_views: int, rank: int, world_size: int) -> List[int]:
    """Indices of the views owned by `rank` (round-robin, so shards differ by <= 1 view)."""
    if world_size <= 0 or not (0 <= rank < world_size):
        raise ValueError(f"bad rank/world_size {rank}/{world_size}")
    return list(range(rank, num_views, world_size))


class GradBuffer:
    """Flat parameter-gradient buffer with per-parameter contiguous views."""

    ORDER = ("means3D", "sh", "opacities", "scales", "rotations")

    def __init__(self, P: int, M: int, device, dtype=torch.float32):
        self.P, self.M = P, M
        sizes = {"means3D": 3 * P, "sh": 3 * M * P, "opacities": P, "scales": 2 * P, "rotations": 4 * P}
        shapes = {"means3D": (P, 3), "sh": (P, M, 3), "opacities": (P, 1), "scales": (P, 2), "rotations": (P, 4)}
        # every segment starts on a 16-byte boundary (the kernel uses vector accesses)
        offs, o = {}, 0
        for k in self.ORDER:
            offs[k] = o
            o += (sizes[k] + 3) // 4 * 4
        self.flat = torch.zeros(o, dtype=dtype, device=device)
        self.views: Dict[str, torch.Tensor] = {
            k: self.flat[offs[k]:offs[k] + sizes[k]].view(*shapes[k]) for k in self.ORDER}

    def zero_(self):
        self.flat.zero_()
        return self

    def all_reduce(self, group=None):
        """The one collective of the view-sharded step: sum of parameter gradients."""
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group)
        return self


def render_views(params: Dict[str, torch.Tensor], settings_list: Sequence[R.GaussianRasterizationSettings],
                 upstream: Optional[Callable[[int, torch.Tensor, torch.Tensor], Tuple[torch.Tensor, torch.Tensor]]],
                 grads: Optional[GradBuffer] = None, view_ids: Optional[Sequence[int]] = None,
                 raster_fn=None, streams: int = 1, cams: Optional[torch.Tensor] = None,
                 upstream_stacked: Optional[Tuple[torch.Tensor, torch.Tensor]] = None):
    """Forward+backward of the given views, accumulating parameter gradients into `grads`.

    params   : dict with contiguous fp32 CUDA tensors means3D [P,3], shs [P,M,3], opacities [P,1],
               scales [P,2], rotations [P,4] (already activated, as LaRa's renderer passes them)
    upstream : callback (view_id, color[3,H,W], allmap[8,H,W]) -> (dL_dcolor, dL_dallmap); this is
               where the caller's loss lives.  Alternatively `upstream_stacked` = (dL_dcolor [V,3,H,W],
               dL_dallmap [V,8,H,W]) when the gradients do not depend on the rendered images.
    cams     : optional pre-packed [V,24] camera records (rasterizer.pack_cameras) of `settings_list`
    streams  : accepted for compatibility, ignored -- all views of the call share ONE launch set
               (every kernel carries a view dimension), which is what multi-streaming approximated
    raster_fn: test hook -- a callable pair replacing (forward_raw, backward_raw), driven view by view
    Returns (list of (color, allmap, radii) per view, grads).
    """
    P = int(params["means3D"].shape[0])
    M = int(params["shs"].shape[1])
    dev = params["means3D"].device
    if grads is None:
        grads = GradBuffer(P, M, dev)
    ids = list(view_ids) if view_ids is not None else list(range(len(settings_list)))
    if len(ids) == 0:
        return [], grads

    if raster_fn is not None or not params["means3D"].is_cuda:
        fwd, bwd = raster_fn if raster_fn is not None else (R.forward_raw, R.backward_raw)
        outs = []
        for vid, rs in zip(ids, settings_list):
            color, allmap, radii, state = fwd(params["means3D"], params["shs"], None, params["opacities"],
                                              params["scales"], params["rotations"], None, rs)
            g_color, g_allmap = upstream(vid, color, allmap)
            bwd(state, radii, params["means3D"], params["shs"], None, params["scales"], params["rotations"], None,
                rs, g_color, g_allmap, out=grads.views, accumulate=True, need_means2D=False)
            outs.append((color, allmap, radii))
        return outs, grads

    from .multiview import shared_view_settings
    settings_list = [R._check_settings(rs, dev) for rs in settings_list]
    H, W, tfx, tfy, deg, prefiltered, debug = shared_view_settings(settings_list)
    if cams is None:
        cams = R.pack_cameras(settings_list, dev)
    color, allmap, radii, state = R.forward_views_raw(
        params["means3D"], params["shs"], None, params["opacities"], params["scales"], params["rotations"], None,
        cams, tfx, tfy, H, W, deg, prefiltered=prefiltered, debug=debug)
    if upstream_stacked is not None:
        g_color, g_allmap = upstream_stacked
    else:
        gs = [upstream(vid, color[k], allmap[k]) for k, vid in enumerate(ids)]
        g_color = torch.stack([g[0] for g in gs]).contiguous()
        g_allmap = torch.stack([g[1] for g in gs]).contiguous()
    R.backward_views_raw(state, radii, params["means3D"], params["shs"], None, params["scales"], params["rotations"],
                         None, cams, tfx, tfy, H, W, deg, g_color, g_allmap, out=grads.views, accumulate=True,
                         need_means2D=False, debug=debug)
    return [(color[k], allmap[k], radii[k]) for k in range(len(ids))], grads
