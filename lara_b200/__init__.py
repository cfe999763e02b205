"""lara_b200 -- H100-native (sm_90a) 2D-Gaussian-surfel rasterizer (drop-in for LaRa's
``diff_surfel_rasterization``).  Importable without a GPU; any use of the rasterizer
requires the in-tree CUDA library ``libsurfel_b200.so`` (``python -m lara_b200.build``)."""
from .rasterizer import (  # noqa: F401
    GaussianRasterizationSettings,
    GaussianRasterizer,
    rasterize_gaussians,
    _RasterizeGaussians,
)
from .coarse_head import CoarseHead  # noqa: F401

__all__ = ["GaussianRasterizationSettings", "GaussianRasterizer", "rasterize_gaussians", "CoarseHead"]
__version__ = "0.1.0"
