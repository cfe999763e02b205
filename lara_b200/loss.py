"""Fused loss -> dL/d(render_img outputs) producer (SURVEY.md 8f rank 3) -- an additional entry point.

LaRa's ``Losses.forward`` (``lightning/loss.py:33-60``) computes, on the ``[H, V*W, C]`` concatenation of a scene's
views, ``mean((image - tar_rgb)^2)`` (+ ``0.5 (1 - MS-SSIM)``) and, after iteration 1000,
``1000 mean(rend_dist) + 0.2 mean((1 - <rend_normal, depth_normal>) acc_map.detach())`` -- ~15 elementwise and
reduction kernels forward, ~20 in autograd, each a full-image HBM round trip, plus the ``torch.cat`` /
``permute`` copies that build the concatenated layout.  ``scene_loss`` computes the same terms directly on the
stacked planar ``[V,C,H,W]`` buffers that ``lara_b200.multiview.render_scene_views`` returns views of: one kernel
for the three sums, one kernel that writes the four gradient maps exactly where the fused epilogue's backward
reads them.  ``ms_ssim=True`` adds LaRa's ``0.5 (1 - MS-SSIM)`` term computed by the fused kernels of
``lara_b200.ssim`` on the planar views read as one ``H x V*W`` image (LaRa's layout); its gradient adds to ``g_image``
through autograd.

``Losses`` is LaRa's ``Losses`` module for the batch renders: all B scenes and both passes in one autograd node, one
loss launch and one MS-SSIM launch set per direction (DESIGN §3.27).
"""
from __future__ import annotations

import ctypes
from typing import Callable, Dict, Optional, Tuple

import torch

from . import _lib
from ._lib import _ptr
from .ssim import _MIN_SIDE, ms_ssim_views


def _planar(t: torch.Tensor) -> torch.Tensor:
    """[V,H,W,C] channel-last view of a planar buffer -> the planar [V,C,H,W] tensor (no copy for the views
    render_scene_views returns)."""
    return t.permute(0, 3, 1, 2).contiguous()


class _SceneLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, rend_normal, depth_normal, rend_dist, acc_map, target, with_reg, batch_scenes):
        dev = image.device
        V, _, H, W = image.shape
        for name, t in (("image", image), ("target", target), ("rend_normal", rend_normal), ("depth_normal", depth_normal),
                        ("rend_dist", rend_dist), ("acc_map", acc_map)):
            if t is None:
                continue
            if not t.is_cuda or t.device != dev or t.dtype != torch.float32 or not t.is_contiguous():
                raise RuntimeError(f"scene_loss: {name} must be a contiguous float32 CUDA tensor on {dev}")
        if tuple(target.shape) != (V, H, W, 3):
            raise RuntimeError(f"scene_loss: tar_rgb must be [V,H,W,3] = {(V, H, W, 3)}, got {tuple(target.shape)}")
        sums = torch.empty(3, dtype=torch.float64, device=dev)
        # partial sums reduced in a fixed order instead of atomics
        ws = (torch.empty(_lib.det_loss_workspace_bytes(_lib.load(), V, H, W) // 8, dtype=torch.float64, device=dev)
              if _lib.deterministic() else None)
        _lib.launch("srf_loss_forward", dev, V, H, W, 1 if with_reg else 0, image.data_ptr(), target.data_ptr(),
                    _ptr(rend_normal), _ptr(depth_normal), _ptr(acc_map), _ptr(rend_dist), sums.data_ptr(), _ptr(ws))
        npx = float(batch_scenes) * V * H * W
        mse = sums[0] / (3.0 * npx)
        dist = sums[1] / npx
        nerr = sums[2] / npx
        loss = mse + (1000.0 * dist + 0.2 * nerr if with_reg else 0.0)
        ctx.save_for_backward(image, target, rend_normal if with_reg else image.new_empty(0),
                              depth_normal if with_reg else image.new_empty(0), acc_map if with_reg else image.new_empty(0))
        ctx.with_reg, ctx.npx = bool(with_reg), npx
        return loss.float(), mse.float(), dist.float(), nerr.float()

    @staticmethod
    def backward(ctx, g_loss, _g_mse, _g_dist, _g_nerr):
        image, target, rn, dn, acc = ctx.saved_tensors
        dev = image.device
        V, _, H, W = image.shape
        up = g_loss.to(torch.float32).contiguous()
        g_image = torch.empty_like(image)
        if ctx.with_reg:
            g_rn, g_dn = torch.empty_like(rn), torch.empty_like(dn)
            g_dist = torch.empty((V, H, W), dtype=torch.float32, device=dev)
        else:
            g_rn = g_dn = g_dist = None
        _lib.launch("srf_loss_backward", dev, V, H, W, 1 if ctx.with_reg else 0, 1.0 / (3.0 * ctx.npx),
                    1000.0 / ctx.npx, 0.2 / ctx.npx, image.data_ptr(), target.data_ptr(),
                    _ptr(rn if ctx.with_reg else None), _ptr(dn if ctx.with_reg else None),
                    _ptr(acc if ctx.with_reg else None), up.data_ptr(), g_image.data_ptr(), _ptr(g_rn), _ptr(g_dn),
                    _ptr(g_dist))
        return g_image, g_rn, g_dn, g_dist, None, None, None, None


def scene_loss(out: Dict[str, torch.Tensor], tar_rgb: torch.Tensor, iter: int, batch_scenes: int = 1,
               ssim: Optional[Callable[[torch.Tensor, torch.Tensor], torch.Tensor]] = None,
               prex: str = "", ms_ssim: bool = False) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """One scene's contribution to ``Losses.forward`` (lightning/loss.py:17-62) from the stacked dict of
    ``render_scene_views`` / ``Renderer.render_views``: ``out[k]`` are ``[V,H,W,C]`` / ``[V,H,W]``, ``tar_rgb`` is the
    batch's ``[V,H,W,3]`` target (``batch['tar_rgb'][i]``).  ``batch_scenes`` = B of the batch (the reference's means run
    over all scenes).
    ``ms_ssim=True`` adds this scene's share of LaRa's MS-SSIM term, ``(0.5 / B) (1 - mean_c value_c)``, with the
    views side by side as one ``H x V*W`` image exactly as LaRa computes it (windows straddle the seams), and sets the
    stat ``ssim`` to ``mean_c value_c / B`` (summed over the scenes: LaRa's stat).
    ``ssim(image[V,3,H,W], target[V,3,H,W]) -> scalar`` adds ``0.5 (1 - ssim)``; it receives the per-view stack, which
    is not LaRa's layout, so the library's MS-SSIM plugged in here gives a different number from LaRa's.
    Returns (loss, scalar_stats) with the reference's stat names."""
    if ms_ssim and ssim is not None:
        raise ValueError("scene_loss: pass either ms_ssim=True or ssim=, not both")
    with_reg = f"rend_dist{prex}" in out and iter > 1000 and prex != "_fine"
    image = _planar(out[f"image{prex}"])
    rn = _planar(out[f"rend_normal{prex}"]) if with_reg else None
    dn = _planar(out[f"depth_normal{prex}"]) if with_reg else None
    dist = out[f"rend_dist{prex}"].contiguous() if with_reg else None
    acc = out[f"acc_map{prex}"].detach().contiguous() if with_reg else None
    loss, mse, distortion, nerr = _SceneLoss.apply(image, rn, dn, dist, acc, tar_rgb.contiguous(), with_reg, int(batch_scenes))
    stats = {f"mse{prex}": mse.detach(), f"psnr{prex}": -10.0 * torch.log10(mse.detach())}
    if ssim is not None:
        s = ssim(image, tar_rgb.permute(0, 3, 1, 2))
        stats[f"ssim{prex}"] = s.detach()
        loss = loss + 0.5 * (1 - s)
    if ms_ssim:
        s = ms_ssim_views(image, tar_rgb.permute(0, 3, 1, 2))
        stats[f"ssim{prex}"] = s.detach() / batch_scenes
        loss = loss + (0.5 / batch_scenes) * (1 - s)
    if with_reg:
        stats[f"distortion{prex}"] = distortion.detach()
        stats[f"normal{prex}"] = nerr.detach()
    return loss, stats


# ---- LaRa's Losses on the batch renders: every scene, both passes ------------------------------------------------------

def _views_addr(t: torch.Tensor) -> _lib.MsSsimAddr:
    """Addressing record of a [B,V,C,H,W] tensor (any strides) read as B images [C, H, V*W], the views side by side."""
    s = t.stride()
    return _lib.MsSsimAddr(s[0], s[2], s[3], s[4], s[1], t.shape[4])


class _BatchLoss(torch.autograd.Function):
    """Both passes of all B scenes in one node: inputs planar [B,V,3,H,W] (image, image_fine or None, rend_normal,
    depth_normal), [B,V,H,W] (rend_dist, acc_map) and the target [B,V,H,W,3].  Returns the fp32 loss, assembled in
    float64 in LaRa's order, and, not differentiable, the loss kernel's sums [3 or 4] (float64) and each pass's MS-SSIM
    mean over (scene, channel) [1 or 2] (float32)."""

    @staticmethod
    def forward(ctx, image, image_fine, rend_normal, depth_normal, rend_dist, acc_map, target, with_reg):
        dev = image.device
        B, V, C, H, W = image.shape
        fine = image_fine is not None
        lib = _lib.load()
        sums = torch.empty(4 if fine else 3, dtype=torch.float64, device=dev)
        ws = (torch.empty(_lib.det_loss_passes_workspace_bytes(lib, B * V, H, W, fine) // 8, dtype=torch.float64,
                          device=dev) if _lib.deterministic() else None)
        _lib.launch("srf_loss_passes_forward", dev, B * V, H, W, 1 if with_reg else 0, image.data_ptr(), _ptr(image_fine),
                    target.data_ptr(), _ptr(rend_normal), _ptr(depth_normal), _ptr(acc_map), _ptr(rend_dist),
                    sums.data_ptr(), _ptr(ws))
        ssim_ws = torch.empty(_lib.ms_ssim_passes_workspace_bytes(lib, B, C, H, V * W, fine), dtype=torch.uint8,
                              device=dev)
        ssim = torch.empty(2 if fine else 1, dtype=torch.float32, device=dev)
        ax, ay = _views_addr(image), _views_addr(target.permute(0, 1, 4, 2, 3))
        _lib.launch("srf_ms_ssim_passes_forward", dev, B, C, H, V * W, image.data_ptr(), _ptr(image_fine),
                    ctypes.byref(ax), target.data_ptr(), ctypes.byref(ay), 1.0, ssim_ws.data_ptr(), ssim.data_ptr())
        loss = assemble_loss(sums, ssim, B * V * H * W, with_reg).float()
        none = image.new_empty(0)
        ctx.save_for_backward(image, image_fine if fine else none, target, rend_normal if with_reg else none,
                              depth_normal if with_reg else none, acc_map if with_reg else none, ssim_ws)
        ctx.fine, ctx.with_reg = fine, bool(with_reg)
        ctx.mark_non_differentiable(sums, ssim)
        return loss, sums, ssim

    @staticmethod
    def backward(ctx, g_loss, _g_sums, _g_ssim):
        image, image_fine, target, rn, dn, acc, ssim_ws = ctx.saved_tensors
        dev = image.device
        B, V, C, H, W = image.shape
        fine, with_reg = ctx.fine, ctx.with_reg
        npx = float(B * V * H * W)
        up = g_loss.to(torch.float32).reshape(1)
        g_image = torch.empty_like(image)
        g_fine = torch.empty_like(image_fine) if fine else None
        if with_reg:
            g_rn, g_dn = torch.empty_like(rn), torch.empty_like(dn)
            g_dist = torch.empty((B, V, H, W), dtype=torch.float32, device=dev)
        else:
            g_rn = g_dn = g_dist = None
        _lib.launch("srf_loss_passes_backward", dev, B * V, H, W, 1 if with_reg else 0, 1.0 / (3.0 * npx),
                    1000.0 / npx, 0.2 / npx, image.data_ptr(), _ptr(image_fine if fine else None), target.data_ptr(),
                    _ptr(rn if with_reg else None), _ptr(dn if with_reg else None), _ptr(acc if with_reg else None),
                    up.data_ptr(), g_image.data_ptr(), _ptr(g_fine), _ptr(g_rn), _ptr(g_dn), _ptr(g_dist))
        # d loss / d ssim of each pass: -0.5 g_loss, as autograd gives it through LaRa's 0.5 * (1 - ssim)
        g_ssim = (up * -0.5).expand(2 if fine else 1).contiguous()
        ax, ay = _views_addr(image), _views_addr(target.permute(0, 1, 4, 2, 3))
        _lib.launch("srf_ms_ssim_passes_backward", dev, B, C, H, V * W, image.data_ptr(),
                    _ptr(image_fine if fine else None), ctypes.byref(ax), target.data_ptr(), ctypes.byref(ay), 1.0,
                    ssim_ws.data_ptr(), g_ssim.data_ptr(), g_image.data_ptr(), _ptr(g_fine), ctypes.byref(ax), 1)
        return g_image, g_fine, g_rn, g_dn, g_dist, None, None, None


def assemble_loss(sums: torch.Tensor, ssim: torch.Tensor, npx: int, with_reg: bool) -> torch.Tensor:
    """LaRa's loss in float64 from the loss kernel's sums and the passes' MS-SSIM values, in LaRa's order:
    mse + 0.5 (1 - ssim) [+ 1000 distortion + 0.2 normal] for the coarse pass, then mse + 0.5 (1 - ssim) for the fine
    pass when ``sums`` has its fourth entry.  ``npx`` = B V H W."""
    s = ssim.to(torch.float64)
    loss = sums[0] / (3.0 * npx) + 0.5 * (1.0 - s[0])
    if with_reg:
        loss = loss + (sums[1] / npx) * 1000.0
        loss = loss + (sums[2] / npx) * 0.2
    if sums.shape[0] > 3:
        loss = loss + sums[3] / (3.0 * npx)
        loss = loss + 0.5 * (1.0 - s[1])
    return loss


_KEYS3 = ("image", "rend_normal", "depth_normal")


class Losses(torch.nn.Module):
    """LaRa's ``Losses`` (``lightning/loss.py``) on the batch renders: ``forward(batch, output, iter) -> (loss,
    scalar_stats)`` with LaRa's rules, names and values, for every scene of the batch and both passes at once.

    ``output`` is ``render_batch_views(...)`` merged with ``render_batch_subset_views(...)``: ``image``,
    ``image_fine`` [B,V,H,W,3], ``acc_map`` [B,V,H,W], ``rend_dist``, ``rend_normal``, ``depth_normal``, ... (the views
    of the planar buffers the renders return, read in place); ``binning*`` and keys no term reads are ignored.
    ``batch['tar_rgb']`` is [B,V,H,W,3].  The fine pass counts when ``acc_map_fine`` is present; the distortion and
    normal terms apply to the coarse pass when ``rend_dist`` is present and ``iter > 1000``.  The stats are detached
    device tensors (nothing is read to the host): ``mse``, ``psnr`` ([1], LaRa's ``-10 log(x) / log(10)``), ``ssim``
    (MS-SSIM over the views side by side, the mean over scenes and channels), ``distortion``, ``normal`` and the fine
    pass's ``mse_fine``, ``psnr_fine``, ``ssim_fine``.  Unlike LaRa's module, an ``output`` without ``image`` raises.
    The forward is one loss launch and one MS-SSIM launch set for both passes; so is the backward."""

    def forward(self, batch, output, iter):
        fn = "Losses"
        if "tar_rgb" not in batch:
            raise KeyError(f"{fn}: batch has no 'tar_rgb'")
        fine = "acc_map_fine" in output
        with_reg = "rend_dist" in output and iter > 1000
        need = ["image"] + (["image_fine"] if fine else []) + (["rend_normal", "depth_normal", "acc_map"] if with_reg else [])
        for k in need:
            if k not in output:
                raise KeyError(f"{fn}: output has no '{k}'")
        tar = batch["tar_rgb"]
        ins = {"tar_rgb": tar, **{k: output[k] for k in need}}
        if with_reg:
            ins["rend_dist"] = output["rend_dist"]
        for k, t in ins.items():
            if not isinstance(t, torch.Tensor):
                raise TypeError(f"{fn}: {k} must be a tensor, got {type(t).__name__}")
            if t.dtype != torch.float32:
                raise TypeError(f"{fn}: {k} must be float32, got {t.dtype}")
        if tar.ndim != 5 or tar.shape[-1] != 3:
            raise ValueError(f"{fn}: tar_rgb must be [B,V,H,W,3], got {tuple(tar.shape)}")
        B, V, H, W = (int(v) for v in tar.shape[:4])
        for k, t in ins.items():
            want = (B, V, H, W) if k in ("rend_dist", "acc_map") else (B, V, H, W, 3)
            if tuple(t.shape) != want:
                raise ValueError(f"{fn}: {k} must be {list(want)} like tar_rgb, got {tuple(t.shape)}")
        if tar.requires_grad:
            raise RuntimeError(f"{fn}: tar_rgb requires grad, but the fused loss gives no gradient for the target; "
                               "detach it")
        if min(H, V * W) <= _MIN_SIDE:
            raise ValueError(f"{fn}: Image size should be larger than {_MIN_SIDE} due to the 4 downsamplings in ms-ssim "
                             f"(H={H}, V*W={V * W})")
        dev = tar.device
        for k, t in ins.items():
            if not t.is_cuda or t.device != dev:
                raise RuntimeError(f"{fn}: {k} must be a CUDA tensor on {dev}, got {t.device}")

        def planar(t):      # [B,V,H,W,3] view of a planar [B*V,3,H,W] buffer -> [B,V,3,H,W] (no copy for those views)
            return t.permute(0, 1, 4, 2, 3).contiguous()
        image = planar(ins["image"])
        image_fine = planar(ins["image_fine"]) if fine else None
        rn = planar(ins["rend_normal"]) if with_reg else None
        dn = planar(ins["depth_normal"]) if with_reg else None
        dist = ins["rend_dist"].contiguous() if with_reg else None
        acc = ins["acc_map"].detach().contiguous() if with_reg else None
        loss, sums, ssim = _BatchLoss.apply(image, image_fine, rn, dn, dist, acc, tar.contiguous(), with_reg)
        npx = float(B * V * H * W)
        ten = torch.full((1,), 10.0, device=dev)
        stats = {}
        for j, prex in enumerate(("", "_fine") if fine else ("",)):
            mse = (sums[3 * j] / (3.0 * npx)).float()
            stats[f"mse{prex}"] = mse
            stats[f"psnr{prex}"] = -10.0 * torch.log(mse) / torch.log(ten)
            stats[f"ssim{prex}"] = ssim[j]
            if with_reg and not j:
                stats["distortion"] = (sums[1] / npx).float()
                stats["normal"] = (sums[2] / npx).float()
        return loss, stats
