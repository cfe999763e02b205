"""Fused MS-SSIM of LaRa's training loss (``lightning/loss.py:15,44-47``: pytorch-msssim 1.0.0
``MS_SSIM(data_range=1.0, size_average=True, channel=3)``) -- an additional entry point, CUDA forward and backward.

The library runs ~10 grouped convolutions and ~20 elementwise kernels per scale over 5 scales, and autograd about twice
that again, each a full-image round trip.  Here each level is one kernel per direction (csrc/ms_ssim.cu) plus one
tiny reduction kernel, and the images are read in place through element strides: a channel-last view such as
LaRa's ``output['image'].permute(0, 3, 1, 2)`` needs no copy.  A maintainer switches LaRa to it by changing one
import in ``lightning/loss.py``::

    from lara_b200.ssim import MS_SSIM          # was: from pytorch_msssim import MS_SSIM

Differences from the library, by design: float32 CUDA inputs only; no gradient for ``Y`` (passing a ``Y`` that requires
grad raises instead of silently dropping it); only LaRa's window (11 taps, sigma 1.5), weights and K.  The per-level
means are reduced in fp64 in a fixed order, so the result is deterministic and at least as accurate as the library's.
"""
from __future__ import annotations

import ctypes

import torch

from . import _lib

_MS_LEVELS = 5
_MIN_SIDE = (11 - 1) * 2 ** (_MS_LEVELS - 1)


def _addr(t: torch.Tensor, views: bool) -> _lib.MsSsimAddr:
    """Addressing record of a [B,C,H,W] tensor (views=False) or of V planar [V,C,H,W] views read as one
    [1,C,H,V*W] image, the views side by side along the width (views=True)."""
    s = t.stride()
    if views:
        return _lib.MsSsimAddr(0, s[1], s[2], s[3], s[0], t.shape[3])
    return _lib.MsSsimAddr(s[0], s[1], s[2], s[3], 0, t.shape[3])


def _logical_shape(t: torch.Tensor, views: bool):
    B, C, H, W = (int(v) for v in t.shape)
    return (1, C, H, B * W) if views else (B, C, H, W)


def check_inputs(fn: str, X: torch.Tensor, Y: torch.Tensor) -> None:
    """The argument checks shared by MS_SSIM and scene_loss(ms_ssim=True), before any launch."""
    for name, t in (("X", X), ("Y", Y)):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{fn}: {name} must be a tensor")
        if t.dtype != torch.float32:
            raise TypeError(f"{fn}: {name} must be float32, got {t.dtype}")
    if X.shape != Y.shape:
        raise ValueError(f"{fn}: Input images should have the same dimensions, but got {tuple(X.shape)} and "
                         f"{tuple(Y.shape)}.")
    if X.ndim != 4:
        raise ValueError(f"{fn}: Input images should be 4-d tensors, but got {tuple(X.shape)}")
    if Y.requires_grad:
        raise RuntimeError(f"{fn}: Y requires grad, but the fused MS-SSIM gives no gradient for the target; detach it")


def _entry(levels: int, what: str, nonnegative_ssim: bool):
    """The C entry srf_ssim_<what> (one level) or srf_ms_ssim_<what> (MS-SSIM's pyramid) and its relu argument;
    MS-SSIM always relu's, so its entries take none."""
    if levels > 1:
        return f"srf_ms_ssim_{what}", ()
    return f"srf_ssim_{what}", (1 if nonnegative_ssim else 0,)


def ssim_launch(dev: torch.device, x_ptr: int, ax, y_ptr: int, ay, shape, data_range: float, size_average: bool,
                nonnegative_ssim: bool, levels: int = 1):
    """The forward (SSIM for levels=1, MS-SSIM for _MS_LEVELS) on logical [B,C,H,W] images at device addresses
    ``x_ptr`` / ``y_ptr`` read through ``ax`` / ``ay``: (out, workspace); the workspace is what the backward needs."""
    B, C, H, W = shape
    nbytes = (_lib.ms_ssim_workspace_bytes if levels > 1 else _lib.ssim_workspace_bytes)(_lib.load(), B, C, H, W)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    out = torch.empty(() if size_average else (B,), dtype=torch.float32, device=dev)
    name, relu = _entry(levels, "forward", nonnegative_ssim)
    _lib.launch(name, dev, B, C, H, W, x_ptr, ctypes.byref(ax), y_ptr, ctypes.byref(ay), float(data_range),
                1 if size_average else 0, *relu, ws.data_ptr(), out.data_ptr())
    return out, ws


class _Ssim(torch.autograd.Function):
    """SSIM (levels=1) or MS-SSIM (levels=_MS_LEVELS) of X against Y, differentiable wrt X."""

    @staticmethod
    def forward(ctx, X, Y, views, data_range, size_average, nonnegative_ssim, levels):
        if not X.is_cuda or Y.device != X.device:
            raise RuntimeError(f"{'MS_SSIM' if levels > 1 else 'ssim'}: X and Y must be CUDA tensors on one device, "
                               f"got {X.device} and {Y.device}")
        shape = _logical_shape(X, views)
        out, ws = ssim_launch(X.device, X.data_ptr(), _addr(X, views), Y.data_ptr(), _addr(Y, views), shape,
                              data_range, size_average, nonnegative_ssim, levels)
        ctx.save_for_backward(X, Y, ws)
        ctx.cfg = (views, float(data_range), bool(size_average), _entry(levels, "backward", nonnegative_ssim), shape)
        return out

    @staticmethod
    def backward(ctx, g_out):
        X, Y, ws = ctx.saved_tensors
        views, data_range, size_average, (name, relu), (B, C, H, W) = ctx.cfg
        up = g_out.to(torch.float32).reshape(-1).contiguous()
        gX = torch.empty_like(X)
        ax, ay, ag = _addr(X, views), _addr(Y, views), _addr(gX, views)
        _lib.launch(name, X.device, B, C, H, W, X.data_ptr(), ctypes.byref(ax), Y.data_ptr(), ctypes.byref(ay),
                    data_range, 1 if size_average else 0, *relu, ws.data_ptr(), up.data_ptr(), gX.data_ptr(),
                    ctypes.byref(ag))
        return gX, None, None, None, None, None, None


def ms_ssim_views(image: torch.Tensor, target: torch.Tensor, data_range: float = 1.0) -> torch.Tensor:
    """MS-SSIM (mean over channels) of V planar views [V,C,H,W] read as one [1,C,H,V*W] image, the views side by side
    along the width as LaRa concatenates them; target as image (any strides, e.g. a permuted [V,H,W,C])."""
    check_inputs("ms_ssim_views", image, target)
    if min(image.shape[2], image.shape[0] * image.shape[3]) <= _MIN_SIDE:
        raise AssertionError(f"Image size should be larger than {_MIN_SIDE} due to the 4 downsamplings in ms-ssim")
    return _Ssim.apply(image, target, True, data_range, True, True, _MS_LEVELS)


class MS_SSIM(torch.nn.Module):
    """Drop-in for ``pytorch_msssim.MS_SSIM`` with the arguments LaRa uses, for 4-D float32 CUDA inputs of any strides.

    ``forward(X, Y)`` returns the mean over (batch, channel) (``size_average=True``) or the per-batch mean over
    channels; differentiable wrt ``X`` only.  Arguments LaRa does not use must keep the library's defaults."""

    def __init__(self, data_range=255, size_average=True, win_size=11, win_sigma=1.5, channel=3, spatial_dims=2,
                 weights=None, K=(0.01, 0.03), win=None):
        super().__init__()
        for name, val, default in (("win_size", win_size, 11), ("win_sigma", win_sigma, 1.5),
                                   ("spatial_dims", spatial_dims, 2), ("K", tuple(K), (0.01, 0.03))):
            if val != default:
                raise ValueError(f"MS_SSIM: {name}={val!r} is not supported (only the default {default!r})")
        if weights is not None and [float(w) for w in weights] != [0.0448, 0.2856, 0.3001, 0.2363, 0.1333]:
            raise ValueError("MS_SSIM: only the default weights are supported")
        if win is not None:
            raise ValueError("MS_SSIM: a custom win is not supported (only the default 11-tap, sigma 1.5 window)")
        self.data_range = data_range
        self.size_average = size_average
        self.channel = int(channel)

    def forward(self, X: torch.Tensor, Y: torch.Tensor) -> torch.Tensor:
        check_inputs("MS_SSIM", X, Y)
        if X.shape[1] != self.channel:
            raise ValueError(f"MS_SSIM: expected {self.channel} channels, got {X.shape[1]}")
        assert min(X.shape[-2:]) > _MIN_SIDE, \
            "Image size should be larger than %d due to the 4 downsamplings in ms-ssim" % _MIN_SIDE
        return _Ssim.apply(X, Y, False, self.data_range, self.size_average, True, _MS_LEVELS)


# ---- single-scale SSIM (pytorch-msssim 1.0.0 ``ssim`` / ``SSIM``) ----------------------------------------------------

def _check_ssim_args(fn: str, win_size, win_sigma, win, K) -> None:
    for name, val, default in (("win_size", win_size, 11), ("win_sigma", win_sigma, 1.5), ("K", tuple(K), (0.01, 0.03))):
        if val != default:
            raise ValueError(f"{fn}: {name}={val!r} is not supported (only the default {default!r})")
    if win is not None:
        raise ValueError(f"{fn}: a custom win is not supported (only the default 11-tap, sigma 1.5 window)")


def _check_ssim_size(fn: str, H: int, W: int) -> None:
    if H < 11 or W < 11:
        raise ValueError(f"{fn}: H and W must be at least the window size 11, got {H} x {W} (pytorch_msssim skips the "
                         "filter along a shorter side with a warning; the fused SSIM does not)")


def ssim(X: torch.Tensor, Y: torch.Tensor, data_range=255, size_average=True, win_size=11, win_sigma=1.5, win=None,
         K=(0.01, 0.03), nonnegative_ssim=False) -> torch.Tensor:
    """Drop-in for ``pytorch_msssim.ssim`` (same signature and defaults) on 4-D float32 CUDA inputs of any strides.

    Returns the mean over (batch, channel) of the per-channel SSIM (``size_average=True``) or the per-batch mean over
    channels; ``nonnegative_ssim`` relu's the per-channel values first.  Differentiable wrt ``X`` only.  H and W must
    be at least 11; arguments other than the library's window and K raise."""
    _check_ssim_args("ssim", win_size, win_sigma, win, K)
    check_inputs("ssim", X, Y)
    _check_ssim_size("ssim", X.shape[2], X.shape[3])
    return _Ssim.apply(X, Y, False, data_range, size_average, nonnegative_ssim, 1)


class SSIM(torch.nn.Module):
    """Drop-in for ``pytorch_msssim.SSIM``: ``forward(X, Y)`` is :func:`ssim` with the module's settings."""

    def __init__(self, data_range=255, size_average=True, win_size=11, win_sigma=1.5, channel=3, spatial_dims=2,
                 K=(0.01, 0.03), nonnegative_ssim=False):
        super().__init__()
        _check_ssim_args("SSIM", win_size, win_sigma, None, K)
        if spatial_dims != 2:
            raise ValueError(f"SSIM: spatial_dims={spatial_dims!r} is not supported (only 2)")
        self.data_range = data_range
        self.size_average = size_average
        self.channel = int(channel)
        self.nonnegative_ssim = nonnegative_ssim

    def forward(self, X: torch.Tensor, Y: torch.Tensor) -> torch.Tensor:
        check_inputs("SSIM", X, Y)
        if X.shape[1] != self.channel:
            raise ValueError(f"SSIM: expected {self.channel} channels, got {X.shape[1]}")
        _check_ssim_size("SSIM", X.shape[2], X.shape[3])
        return _Ssim.apply(X, Y, False, self.data_range, self.size_average, self.nonnegative_ssim, 1)


def ssim_views(image: torch.Tensor, target: torch.Tensor, data_range: float = 1.0, view_range=None) -> torch.Tensor:
    """SSIM (mean over channels) of V planar views [V,C,H,W] read as one [1,C,H,V*W] image, the views side by side
    along the width as LaRa concatenates them (evaluation.py:93); target as image (any strides, e.g. a permuted
    [V,H,W,C]).  ``view_range`` (v0, v1) keeps views v0 .. v1 - 1 of both, as ``eval_novel_view_only`` does."""
    if view_range is not None:
        v0, v1 = (int(v) for v in view_range)
        if not 0 <= v0 < v1 <= image.shape[0]:
            raise ValueError(f"ssim_views: view range [{v0}, {v1}) is empty or outside the {image.shape[0]} views")
        image, target = image[v0:v1], target[v0:v1]
    check_inputs("ssim_views", image, target)
    _check_ssim_size("ssim_views", image.shape[2], image.shape[0] * image.shape[3])
    return _Ssim.apply(image, target, True, data_range, True, False, 1)
