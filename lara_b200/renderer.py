"""A faster ``Renderer`` with the interface of LaRa's ``lightning/renderer_2dgs.Renderer``.

The reference class does three things per view: activations (``renderer_2dgs.py:183-188``), the
rasterizer call (``:209-218``) and ~12 torch ops of post-processing (``:220-268``).  This class
keeps the constructor, ``set_bg_color``, ``set_rasterizer`` and the ``render_img`` signature /
returned dict, but runs this package's rasterizer and the fused epilogue (``lara_b200.epilogue``).  It is
an *additional* entry point: LaRa's own ``renderer_2dgs.py`` keeps working unchanged on top of the
drop-in ``diff_surfel_rasterization`` package; a maintainer who wants the fused epilogue's saving per view
replaces ``from lightning.renderer_2dgs import Renderer`` by ``from lara_b200.renderer import Renderer``.
"""
from __future__ import annotations

import math

import torch
from torch import nn

from .epilogue import render_img_epilogue
from .rasterizer import GaussianRasterizationSettings, GaussianRasterizer


class Renderer(nn.Module):
    def __init__(self, sh_degree: int = 3, white_background: bool = True, radius: float = 1,
                 fused_activations: bool = True):
        super().__init__()
        # True: sigmoid / exp / normalize and their vjps run inside the preprocess kernels (SURVEY 8f rank 1)
        self.fused_activations = fused_activations
        self.sh_degree = sh_degree
        self.white_background = white_background
        self.radius = radius
        self.bg_color = torch.tensor([1, 1, 1] if white_background else [0, 0, 0], dtype=torch.float32)
        # activations of the reference (renderer_2dgs.py:106-114)
        self.scaling_activation = torch.exp
        self.opacity_activation = torch.sigmoid
        self.rotation_activation = torch.nn.functional.normalize

    def set_bg_color(self, bg):
        self.bg_color = bg

    def set_rasterizer(self, viewpoint_camera, scaling_modifier: float = 1.0, device="cuda"):
        settings = GaussianRasterizationSettings(
            image_height=int(viewpoint_camera.image_height),
            image_width=int(viewpoint_camera.image_width),
            tanfovx=math.tan(viewpoint_camera.FoVx * 0.5),
            tanfovy=math.tan(viewpoint_camera.FoVy * 0.5),
            bg=self.bg_color.to(device),
            scale_modifier=scaling_modifier,
            viewmatrix=viewpoint_camera.world_view_transform,
            projmatrix=viewpoint_camera.full_proj_transform,
            sh_degree=self.sh_degree,
            campos=viewpoint_camera.camera_center,
            prefiltered=False,
            debug=False,
        )
        return GaussianRasterizer(raster_settings=settings)

    def render_img(self, cam, rays, centers, shs, opacity, scales, rotations, device, cov3D_precomp=None,
                   prex: str = "", depth_ratio: float = 0.0):
        rasterizer = self.set_rasterizer(cam, device=device)
        fuse = self.fused_activations and cov3D_precomp is None and scales is not None and rotations is not None
        if not fuse:
            opacity = self.opacity_activation(opacity)
            if scales is not None:
                scales = self.scaling_activation(scales)
            if rotations is not None:
                rotations = self.rotation_activation(rotations)
        # gradient sink for the screen-space statistic, as in the reference (:193-206)
        screenspace_points = torch.zeros_like(centers, dtype=centers.dtype, requires_grad=True, device=device) + 0
        try:
            screenspace_points.retain_grad()
        except Exception:
            pass
        if fuse:
            rendered_image, radii, allmap = rasterizer.forward_raw_activations(
                means3D=centers, means2D=screenspace_points, shs=shs, opacities=opacity, scales=scales,
                rotations=rotations)
        else:
            rendered_image, radii, allmap = rasterizer(
                means3D=centers, means2D=screenspace_points, shs=shs, opacities=opacity, scales=scales,
                rotations=rotations, cov3D_precomp=cov3D_precomp)
        if rays is None:
            return rendered_image.clamp(0, 1)
        return render_img_epilogue(rendered_image, allmap, rays, cam.world_view_transform, depth_ratio, prex)

    def render_views(self, cams, rays, centers, shs, opacity, scales, rotations, device, bg_colors=None,
                     prex: str = "", depth_ratio: float = 0.0, streams: int = 3, keep_binning: bool = False):
        """All target views of one scene in one autograd node (the loop of network.py:486-495):
        ``cams`` a sequence of MiniCam-like objects, ``rays`` [V,H,W,6] (or None), ``bg_colors`` an
        optional [V,3] / sequence of per-view backgrounds (network.py:489-490), default ``self.bg_color``.
        Returns stacked ``{key: [V,H,W,C]}``; ``lara_b200.multiview.concat_views`` gives network.py:525's layout.
        ``keep_binning``: also ``out["binning"+prex]``, from which :meth:`render_subset_views` renders the fine pass."""
        from .multiview import render_scene_views
        settings = []
        for j, cam in enumerate(cams):
            if bg_colors is not None:
                self.set_bg_color(bg_colors[j])
            settings.append(self.set_rasterizer(cam, device=device).raster_settings)
        fuse = self.fused_activations
        if not fuse:
            opacity = self.opacity_activation(opacity)
            scales = self.scaling_activation(scales)
            rotations = self.rotation_activation(rotations)
        return render_scene_views(centers, shs, opacity, scales, rotations, settings, rays=rays, depth_ratio=depth_ratio,
                                  raw_activations=fuse, streams=streams, prex=prex, keep_binning=keep_binning)

    def render_subset_views(self, binning, mask, shs_fine, prex: str = "_fine"):
        """The fine pass over ``mask`` of the Gaussians a ``render_views(..., keep_binning=True)`` call rendered, with
        the SH coefficients ``shs_fine``: ``lara_b200.multiview.render_subset_views``."""
        from .multiview import render_subset_views
        return render_subset_views(binning, mask, shs_fine, prex=prex)

    def render_batch_views(self, cams, rays, centers, shs, opacity, scales, rotations, device, bg_colors=None,
                           prex: str = "", depth_ratio: float = 0.0, keep_binning: bool = False):
        """:meth:`render_views` for all B scenes of a batch in one launch set: ``cams[b]`` scene b's V cameras,
        ``rays`` [B,V,H,W,6] (or None), Gaussian tensors [B,P,...], ``bg_colors[b][j]`` optional per-view backgrounds.
        Returns ``{key: [B,V,H,W,C]}`` (``lara_b200.multiview.render_batch_views``)."""
        from .multiview import render_batch_views
        settings = []
        for b, scene_cams in enumerate(cams):
            row = []
            for j, cam in enumerate(scene_cams):
                if bg_colors is not None:
                    self.set_bg_color(bg_colors[b][j])
                row.append(self.set_rasterizer(cam, device=device).raster_settings)
            settings.append(row)
        fuse = self.fused_activations
        if not fuse:
            opacity = self.opacity_activation(opacity)
            scales = self.scaling_activation(scales)
            rotations = self.rotation_activation(rotations)
        return render_batch_views(centers, shs, opacity, scales, rotations, settings, rays=rays, depth_ratio=depth_ratio,
                                  raw_activations=fuse, prex=prex, keep_binning=keep_binning)

    def render_batch_subset_views(self, binning, masks, shs_fine, prex: str = "_fine"):
        """The fine pass of all scenes of a :meth:`render_batch_views` call with ``keep_binning=True``, ``masks`` [B,P]
        bool or their ``lara_b200.multiview.FineSubset``: ``lara_b200.multiview.render_batch_subset_views``."""
        from .multiview import render_batch_subset_views
        return render_batch_subset_views(binning, masks, shs_fine, prex=prex)
