"""Per-scene refinement of LaRa's predicted Gaussians: the ``finetuning`` block of ``configs/infer.yaml`` with the
parameter groups of ``Renderer.get_params`` (``lightning/renderer_2dgs.py:142-152``).

* :class:`GaussianAdam` -- ``torch.optim.Adam`` over get_params' six groups (xyz, f_dc, f_rest, opacity, scaling,
  rotation) as one launch per step (``srf_gaussian_adam_step``, csrc/finetune.cu), on the five tensors of the Gaussian
  record as they are: f_dc and f_rest are the first and the remaining coefficients of one ``shs`` tensor, which
  ``torch.optim.Adam`` cannot put in two groups without splitting it into two leaves.
* :func:`finetune_scene` -- the refinement loop: the scene's source views rendered in one launch set
  (``Renderer.render_views``), LaRa's training loss after iteration 1000 (``scene_loss(..., ms_ssim=True)``), one Adam
  step; no host read inside the loop.
* :func:`sample_cameras` -- ``MiniCam``-equivalent cameras of a sample's target views.
* :func:`finetune_settings` -- the loop's arguments from LaRa's ``cfg.infer.finetuning``.
"""
from __future__ import annotations

import ctypes
from typing import Dict, Mapping, Sequence, Tuple

import torch

from . import _lib
from .loss import scene_loss
from .scene import PathCamera

GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")     # include/surfel_finetune.h SRF_ADAM_*
SH_COEFFS = (1, 4, 9, 16)
LR_KEYS = ("position_lr", "feature_lr", "opacity_lr", "scaling_lr", "rotation_lr")
# scene_loss adds the distortion and normal-consistency terms for iterations past 1000 (lightning/loss.py:50)
_REGULARISED_ITER = 1001


def group_lrs(position_lr: float, feature_lr: float, opacity_lr: float, scaling_lr: float,
              rotation_lr: float) -> Tuple[float, ...]:
    """The learning rates of get_params' groups, in :data:`GROUPS` order: f_rest at ``feature_lr / 20``."""
    return (float(position_lr), float(feature_lr), feature_lr / 20.0, float(opacity_lr), float(scaling_lr),
            float(rotation_lr))


def finetune_settings(finetuning: Mapping) -> Dict:
    """``steps`` and the five learning rates of LaRa's ``cfg.infer.finetuning`` (a dict or an OmegaConf node), as the
    keyword arguments of :func:`finetune_scene`.  ``with_ft`` is the caller's switch and is not part of them."""
    out = {"steps": int(finetuning["steps"])}
    out.update({k: float(finetuning[k]) for k in LR_KEYS})
    return out


class GaussianAdam:
    """``torch.optim.Adam(get_params(...), betas, eps)`` over the Gaussian record ``centers [n,3]``, ``shs [n,M,3]``,
    ``opacity [n,1]``, ``scaling [n,2]``, ``rotation [n,4]`` (contiguous fp32 CUDA leaves, updated in place).

    Each :meth:`step` is one launch that reads every ``.grad``, updates the parameters and both moments with torch's
    single-tensor arithmetic, and zeroes the gradients (so the next backward accumulates into zeros, as after
    ``zero_grad(set_to_none=False)``).  Betas and eps default to those of the 3DGS ``training_setup`` that get_params
    comes from.  The object owns the moments (fp32, ``2 n (10 + 3 M)`` values) and the step count."""

    def __init__(self, centers: torch.Tensor, shs: torch.Tensor, opacity: torch.Tensor, scaling: torch.Tensor,
                 rotation: torch.Tensor, position_lr: float, feature_lr: float, opacity_lr: float, scaling_lr: float,
                 rotation_lr: float, betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-15):
        self.params = (centers, shs, opacity, scaling, rotation)
        n = int(centers.shape[0]) if centers.ndim == 2 else -1
        M = int(shs.shape[1]) if shs.ndim == 3 else -1
        shapes = ((n, 3), (n, M, 3), (n, 1), (n, 2), (n, 4))
        dev = centers.device
        for name, t, shape in zip(("centers", "shs", "opacity", "scaling", "rotation"), self.params, shapes):
            if (not t.is_cuda or t.device != dev or t.dtype != torch.float32 or not t.is_contiguous()
                    or tuple(t.shape) != shape):
                raise ValueError(f"GaussianAdam: {name} must be a contiguous float32 CUDA tensor of shape {shape} on "
                                 f"{dev}, got {t.dtype} {tuple(t.shape)} on {t.device}")
        if M not in SH_COEFFS:
            raise ValueError(f"GaussianAdam: shs has {M} coefficients, not one of {SH_COEFFS}")
        self.n, self.M, self.device = n, M, dev
        self.lr = group_lrs(position_lr, feature_lr, opacity_lr, scaling_lr, rotation_lr)
        self.betas = (float(betas[0]), float(betas[1]))
        self.eps = float(eps)
        self.moments = torch.zeros(2 * n * (10 + 3 * M), dtype=torch.float32, device=dev)
        self.step_count = 0

    def exp_avg(self) -> Tuple[torch.Tensor, ...]:
        """Views of the first moment, shaped as the five parameters."""
        return self._split(self.moments[: self.moments.numel() // 2])

    def exp_avg_sq(self) -> Tuple[torch.Tensor, ...]:
        """Views of the second moment, shaped as the five parameters."""
        return self._split(self.moments[self.moments.numel() // 2:])

    def _split(self, flat: torch.Tensor) -> Tuple[torch.Tensor, ...]:
        out, off = [], 0
        for p in self.params:
            out.append(flat[off:off + p.numel()].view(p.shape))
            off += p.numel()
        return tuple(out)

    @torch.no_grad()
    def step(self) -> None:
        grads = []
        for name, p in zip(("centers", "shs", "opacity", "scaling", "rotation"), self.params):
            g = p.grad
            if g is None or g.dtype != torch.float32 or g.shape != p.shape or not g.is_contiguous() or g.device != p.device:
                raise RuntimeError(f"GaussianAdam.step: {name} needs a contiguous float32 gradient of its own shape")
            grads.append(g)
        self.step_count += 1
        t = float(self.step_count)
        beta1, beta2 = self.betas
        bc1 = 1 - beta1 ** t                       # torch's fp64 host arithmetic, to the operation
        bc2_sqrt = (1 - beta2 ** t) ** 0.5
        _lib.launch("srf_gaussian_adam_step", self.device, self.n, self.M,
                    (ctypes.c_void_p * 5)(*(p.data_ptr() for p in self.params)),
                    (ctypes.c_void_p * 5)(*(g.data_ptr() for g in grads)), self.moments.data_ptr(),
                    (ctypes.c_double * 6)(*self.lr), beta1, beta2, self.eps, bc1, bc2_sqrt, 1)


def sample_cameras(sample: Mapping, views: Sequence[int]) -> list:
    """``PathCamera``s of scene 0's target views ``views``, built as LaRa's ``MiniCam(c2w, W, H, fovy, fovx, znear, zfar)``
    (lightning/network.py:476-492) from ``tar_c2w``, ``fovx``, ``fovy`` and ``near_far``, and moved to the device of
    ``tar_rgb``.  The matrices are computed on the host in fp32, so they may differ from MiniCam's device-side inverse
    in the last bits."""
    tar = sample["tar_rgb"]
    H, W = int(tar.shape[2]), int(tar.shape[3])
    c2w = sample["tar_c2w"][0].detach().to("cpu", torch.float32)
    znear, zfar = (float(x) for x in sample["near_far"][0].detach().cpu().reshape(2))
    fovx, fovy = float(sample["fovx"][0]), float(sample["fovy"][0])
    cams = []
    for j in views:
        cam = PathCamera(c2w[int(j)], H, W, fovx, znear, zfar, fovy=fovy)
        cam.to_device(tar.device)
        cams.append(cam)
    return cams


def finetune_scene(renderer, gs_params, sample: Mapping, n_views: int, steps: int, position_lr: float,
                   feature_lr: float, opacity_lr: float, scaling_lr: float, rotation_lr: float):
    """Refine LaRa's fine Gaussians of scene 0 on its ``n_views`` source views for ``steps`` steps.

    ``renderer`` is a ``lara_b200.renderer.Renderer``; ``gs_params`` LaRa's fine ``render_pkg[1]``:
    ``(centers[mask] [n,3], shs_fine [n,M,3], opacity [P,1], scaling [P,2], rotation [P,4], mask [P])`` with raw
    (pre-activation) opacity, scaling and rotation.  Only the source views ``tar_c2w``, ``tar_rgb``, ``tar_rays``,
    ``bg_color`` and ``near_far`` at ``[0, :n_views]`` and ``fovx`` / ``fovy`` are read; the novel views are never
    touched.  Each step renders the source views in one launch set, takes LaRa's loss after iteration 1000 (MSE,
    ``0.5 (1 - MS-SSIM)`` on the views side by side, ``1000`` distortion and ``0.2`` normal consistency) and one
    :class:`GaussianAdam` step with get_params' groups.

    Returns ``(refined gs_params, losses)``: the tuple has ``gs_params``' structure, with the rows of opacity, scaling
    and rotation outside ``mask`` unchanged bit for bit, and ``losses`` is a device tensor [steps] of each step's loss
    before its update.  Runs with gradients whatever the caller's grad mode (``torch.no_grad()`` and
    ``torch.inference_mode()`` included) on fresh copies of the inputs; the renderer's background is restored."""
    centers, shs, opacity, scaling, rotation, mask = gs_params
    steps, n_views = int(steps), int(n_views)
    if steps < 0 or n_views <= 0:
        raise ValueError(f"finetune_scene: steps = {steps} and n_views = {n_views} must be >= 0 and > 0")
    dev = centers.device
    bg_saved = renderer.bg_color
    with torch.inference_mode(False), torch.enable_grad():
        leaves = [t.detach().clone().contiguous().requires_grad_(True)
                  for t in (centers, shs, opacity[mask], scaling[mask], rotation[mask])]
        cams = sample_cameras(sample, range(n_views))
        rays = sample["tar_rays"][0, :n_views].clone()
        tar = sample["tar_rgb"][0, :n_views].clone()
        bg = sample["bg_color"][0, :n_views].clone()
        opt = GaussianAdam(*leaves, position_lr, feature_lr, opacity_lr, scaling_lr, rotation_lr)
        losses = torch.empty(steps, dtype=torch.float32, device=dev)
        try:
            for i in range(steps):
                out = renderer.render_views(cams, rays, *leaves, dev, bg_colors=bg)
                loss, _ = scene_loss(out, tar, _REGULARISED_ITER, batch_scenes=1, ms_ssim=True)
                loss.backward()
                losses[i] = loss.detach()
                opt.step()
        finally:
            renderer.set_bg_color(bg_saved)
        refined = []
        for full, new in zip((opacity, scaling, rotation), leaves[2:]):
            t = full.detach().clone()
            t[mask] = new.detach()
            refined.append(t)
    return (leaves[0].detach(), leaves[1].detach(), *refined, mask), losses
