"""LaRa's per-scene evaluation on the GPU (``evaluation.py:83-141``): the novel-view metrics and the turntable video.

* :func:`novel_view_metrics` -- PSNR, SSIM (pytorch-msssim 1.0.0 ``ssim``) and, with ``eval_depth``, the masked depth
  error and threshold accuracies, under LaRa's names.  One kernel computes every sum in a fixed-order fp64 reduction
  (csrc/eval.cu), the fused SSIM reads the same views in place, and the only host transfer is the final scalars.
* :func:`video_path` -- LaRa's turntable cameras (``tools/gen_video_path.py:uni_video_path``) as ``PathCamera``s.
* :func:`video_frames` / :func:`render_video_frames` -- the uint8 RGB and normal frames LaRa writes with
  ``imageio.mimwrite``, rendered forward-only in chunks of views and quantised on the device.

LPIPS (pretrained VGG / AlexNet weights), the Mitsuba mesh video, the ``unposed`` path and the preview grid stay with
LaRa (DESIGN §8).
"""
from __future__ import annotations

import ctypes
import math
from typing import Dict, Optional, Sequence

import numpy as np
import torch

from . import _lib
from .scene import PathCamera
from .ssim import _check_ssim_size, ssim_launch


def _addr_views(t: torch.Tensor, V: int, H: int, W: int, C: int, what: str) -> _lib.MsSsimAddr:
    """Addressing record of a tensor holding V views of H x W x C, read as one logical [1,C,H,V*W] image.  Accepted
    layouts: LaRa's concatenated [H, V*W, C] (an optional leading 1; C = 1 may be absent), a per-view stack
    [V,H,W,C] (C = 1 may be absent) and planar views [V,C,H,W]; any strides."""
    shape = tuple(int(s) for s in t.shape)
    if len(shape) == 4 and shape[0] == 1 and shape[1:] in ((H, V * W, C),) and (V, H, W, C) != shape:
        shape, t = shape[1:], t[0]
    if C == 1 and len(shape) >= 3 and shape[-1] == 1 and shape not in ((V, C, H, W),):
        shape, t = shape[:-1], t[..., 0]
        if len(shape) == 3 and shape[0] == 1 and shape[1:] == (H, V * W):
            shape, t = shape[1:], t[0]
    s = t.stride()
    if C == 1 and shape == (V, H, W):
        return _lib.MsSsimAddr(0, 0, s[1], s[2], s[0], W)
    if C == 1 and shape == (H, V * W):
        return _lib.MsSsimAddr(0, 0, s[0], s[1], 0, V * W)
    if shape == (V, H, W, C):
        return _lib.MsSsimAddr(0, s[3], s[1], s[2], s[0], W)
    if shape == (V, C, H, W):
        return _lib.MsSsimAddr(0, s[1], s[2], s[3], s[0], W)
    if shape == (H, V * W, C):
        return _lib.MsSsimAddr(0, s[2], s[0], s[1], 0, V * W)
    raise ValueError(f"novel_view_metrics: {what} of shape {tuple(t.shape)} is none of [H, V*W, {C}], [V,H,W,{C}] or "
                     f"[V,{C},H,W] for V={V}, H={H}, W={W}")


def _check_tensor(t, what: str, device, dtype=torch.float32) -> torch.Tensor:
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"novel_view_metrics: {what} must be a tensor")
    if t.device != device:
        raise RuntimeError(f"novel_view_metrics: {what} is on {t.device}, expected {device}")
    if dtype is not None and t.dtype != dtype:
        raise TypeError(f"novel_view_metrics: {what} must be {dtype}, got {t.dtype}")
    return t


@torch.no_grad()
def novel_view_metrics(out: Dict[str, torch.Tensor], sample: Dict, n_views: int, eval_novel_view_only: bool = True,
                       eval_depth: Sequence[float] = (), image_key: str = "image_fine",
                       depth_key: str = "depth_fine") -> Dict:
    """LaRa's per-scene numbers (evaluation.py:83-111) for the first scene of ``sample``:

    ``{"psnr": -10 log10(mean squared error), "ssim": ssim(images, img_gt, data_range=1.0)}`` over the target views
    ``n_views ..`` (``eval_novel_view_only``) or all of them, both None when that range is empty (LaRa then records
    nothing); with ``eval_depth`` also ``"depth_acc": [mean |d - d_gt| over tar_msk, acc(threshold) ...]`` over all
    views, NaN for an empty mask.

    ``out[image_key]`` / ``out[depth_key]`` are LaRa's concatenated ``[1, H, V*W, C]`` outputs or this package's
    per-view ``[V,H,W,C]`` / planar ``[V,C,H,W]`` renders; ``sample`` holds ``tar_rgb [B,V,H,W,3]`` and, for depth,
    ``tar_dep`` and ``tar_msk`` ``[B,V,H,W]``."""
    thresholds = [float(t) for t in eval_depth]
    if len(thresholds) > 8:
        raise ValueError(f"novel_view_metrics: at most 8 depth thresholds, got {len(thresholds)}")
    tar = sample["tar_rgb"][0]
    if tar.ndim != 4 or tar.shape[-1] != 3:
        raise ValueError(f"novel_view_metrics: tar_rgb[0] must be [V,H,W,3], got {tuple(tar.shape)}")
    V, H, W = (int(s) for s in tar.shape[:3])
    image = out[image_key]
    dev = image.device
    if not image.is_cuda:
        raise RuntimeError("novel_view_metrics: the renders must be CUDA tensors")
    _check_tensor(image, image_key, dev)
    _check_tensor(tar, "tar_rgb", dev)
    v0 = min(int(n_views), V) if eval_novel_view_only else 0
    ai, at = _addr_views(image, V, H, W, 3, image_key), _addr_views(tar, V, H, W, 3, "tar_rgb")
    lib = _lib.load()
    depth = dgt = msk = None
    ad = ag = am = None
    with_depth = len(thresholds) > 0
    if with_depth:
        depth = _check_tensor(out[depth_key], depth_key, dev)
        dgt = _check_tensor(sample["tar_dep"][0], "tar_dep", dev)
        msk = _check_tensor(sample["tar_msk"][0], "tar_msk", dev, None)
        if msk.dtype not in (torch.bool, torch.uint8):
            msk = msk != 0                     # .bool(): nonzero (NaN included) is inside
        ad, ag, am = (_addr_views(t, V, H, W, 1, k) for t, k in ((depth, depth_key), (dgt, "tar_dep"), (msk, "tar_msk")))
    ws = torch.empty(_lib.eval_workspace_bytes(lib), dtype=torch.uint8, device=dev)
    n_out = 3 + len(thresholds)
    res = torch.empty(n_out + 1, dtype=torch.float64, device=dev)
    thr = (ctypes.c_double * max(1, len(thresholds)))(*thresholds)
    _lib.launch("srf_eval_metrics", dev, V, H, W, v0, V, image.data_ptr(), ctypes.byref(ai), tar.data_ptr(),
                ctypes.byref(at), _lib._ptr(depth), ctypes.byref(ad) if with_depth else None, _lib._ptr(dgt),
                ctypes.byref(ag) if with_depth else None, _lib._ptr(msk), ctypes.byref(am) if with_depth else None,
                len(thresholds), thr, ws.data_ptr(), res.data_ptr())
    width = (V - v0) * W
    if width > 0:
        _check_ssim_size("novel_view_metrics", H, width)
        s, _ = ssim_launch(dev, _view_ptr(image, ai, v0, W), ai, _view_ptr(tar, at, v0, W), at, (1, 3, H, width),
                           1.0, True, False)
        res[n_out:].copy_(s.reshape(1))
    vals = res.tolist()                        # the one host transfer
    m = {"psnr": None, "ssim": None}
    if width > 0:
        m["psnr"] = -10.0 * math.log10(vals[0] / (3.0 * H * width))
        m["ssim"] = float(np.float32(vals[n_out]))
    if with_depth:
        cnt = vals[2]
        m["depth_acc"] = [vals[1] / cnt if cnt else float("nan")] + \
                         [vals[3 + t] / cnt if cnt else float("nan") for t in range(len(thresholds))]
    return m


def _view_ptr(t: torch.Tensor, a: _lib.MsSsimAddr, v0: int, W: int) -> int:
    """Address of column v0 * W of the logical image ``a`` reads from ``t``: read through the same record from there,
    the columns of views v0 .. form an image of their own."""
    return t.data_ptr() + t.element_size() * v0 * (a.sv if a.sv else W * a.sx)


# ---- turntable video ------------------------------------------------------------------------------------------------

_GOBJ_C2W = ([[0, 1.0, 0.0], [0.4515947, 0.0, -0.8922232], [-0.8922232, 0, -0.4515947]], [1.70006549, 0.0, 0.8604804])
_I3D_C2W = ([[-7.0710677e-01, 2.4184476e-01, -6.6446304e-01],
             [7.0710677e-01, 2.4184476e-01, -6.6446304e-01],
             [-5.2163419e-17, -9.3969262e-01, -3.4202015e-01]], [1.328926, 1.328926, 6.8404031e-01])
_I3D_TRANSFORM = [[-7.0710677e-01, 7.0710677e-01, 7.8504622e-17, 0.0000000e+00],
                  [2.4184476e-01, 2.4184476e-01, -9.3969262e-01, 0.0000000e+00],
                  [-6.6446304e-01, -6.6446304e-01, -3.4202015e-01, 0.0000000e+00],
                  [0.0000000e+00, 0.0000000e+00, 0.0000000e+00, 1.0000000e+00]]


def _rot4(axis: str, angle: float) -> torch.Tensor:
    from scipy.spatial.transform import Rotation
    m = torch.eye(4)
    m[:3, :3] = torch.tensor(Rotation.from_euler(axis, angle).as_matrix())
    return m


def video_path(N: int, dataset_name: str, img_size, sample: Optional[Dict] = None, fov=None,
               elevation: float = 0) -> list:
    """LaRa's turntable path (``uni_video_path(N, cfg.infer.dataset, sample, fov)``): N ``PathCamera``s whose matrices
    equal those of LaRa's ``MiniCam``s, built with the same fp32 CPU operations.  ``img_size`` is (width, height),
    ``fov`` (fovx, fovy) as floats or one-element tensors.  LaRa's quirks are kept: the ``gobjeverse`` / ``GSO`` path
    always uses a field of view of 0.75 whatever ``fov`` says, and both paths apply ``sample['transform_mats'][0]``.
    The ``unposed`` path (spline interpolation of the target poses) is not restated."""
    width, height = (int(s) for s in img_size)
    if dataset_name in ("gobjeverse", "GSO"):
        znear, zfar, axis = 0.5, 2.5, "y"
        fovx = fovy = 0.75                     # sic: LaRa overrides the fov it was given
        rot, pos = _GOBJ_C2W
        transform = torch.eye(4) if sample is None else sample["transform_mats"][0].cpu().squeeze(0)
    elif dataset_name in ("instant3d", "mvgen"):
        znear, zfar, axis = 1.0, 3.0, "x"
        fovx, fovy = (0.7, 0.7) if fov is None else (float(fov[0]), float(fov[1]))
        rot, pos = _I3D_C2W
        transform = torch.tensor(_I3D_TRANSFORM) if sample is None else sample["transform_mats"][0].cpu().squeeze(0)
    elif dataset_name == "unposed":
        raise NotImplementedError("video_path: the unposed path (spline interpolation of the target poses) is not "
                                  "restated; use LaRa's tools/gen_video_path.py")
    else:
        raise ValueError(f"video_path: unknown dataset {dataset_name!r}")
    c2w = torch.eye(4)
    c2w[:3, :3] = torch.tensor(rot).t() if axis == "y" else torch.tensor(rot)
    c2w[:3, 3] = torch.tensor(pos)
    c2w = _rot4(axis, elevation / 180.0 * math.pi) @ c2w
    step = _rot4("z", math.pi * 2 / N)
    cams = [PathCamera(transform @ c2w, height, width, fovx, znear, zfar, fovy=fovy)]
    for _ in range(N - 1):
        c2w = step @ c2w
        cams.append(PathCamera(transform @ c2w, height, width, fovx, znear, zfar, fovy=fovy))
    return cams


def video_frames(image: torch.Tensor, normal: Optional[torch.Tensor] = None, alpha: Optional[torch.Tensor] = None,
                 out_rgb: Optional[torch.Tensor] = None, out_nrm: Optional[torch.Tensor] = None):
    """uint8 frames [N,H,W,3] of renders ``image`` / ``normal`` [N,H,W,3] and ``alpha`` [N,H,W] (any strides, fp32,
    CUDA), rounded as LaRa rounds them (evaluation.py:132-136): ``round(image*255)`` and
    ``round((((normal*alpha + 1 - alpha) + 1)/2)*255)``.  Values outside [0, 255] saturate and NaN gives 0.
    Returns (rgb, nrm); nrm is None without ``normal``.  ``out_rgb`` / ``out_nrm`` receive the frames when given."""
    if image.ndim != 4 or image.shape[-1] != 3 or image.dtype != torch.float32 or not image.is_cuda:
        raise ValueError(f"video_frames: image must be a CUDA float32 [N,H,W,3], got {image.dtype} {tuple(image.shape)}")
    N, H, W = (int(s) for s in image.shape[:3])
    dev = image.device

    def addr(t, C):
        if t.dtype != torch.float32 or t.device != dev or tuple(t.shape[:3]) != (N, H, W):
            raise ValueError(f"video_frames: expected CUDA float32 [{N},{H},{W}{',3' if C == 3 else ''}], got "
                             f"{t.dtype} {tuple(t.shape)} on {t.device}")
        s = t.stride()
        return _lib.MsSsimAddr(s[0], s[3] if C == 3 else 0, s[1], s[2], 0, W)

    def frames(o):
        if o is None:
            return torch.empty((N, H, W, 3), dtype=torch.uint8, device=dev)
        if o.dtype != torch.uint8 or tuple(o.shape) != (N, H, W, 3) or not o.is_contiguous() or o.device != dev:
            raise ValueError(f"video_frames: output must be a contiguous CUDA uint8 [{N},{H},{W},3]")
        return o

    ai = addr(image, 3)
    rgb = frames(out_rgb)
    nrm = an = aa = None
    if normal is not None:
        if alpha is None:
            raise ValueError("video_frames: normal frames need alpha")
        if alpha.ndim == 4 and alpha.shape[-1] == 1:
            alpha = alpha[..., 0]
        an, aa = addr(normal, 3), addr(alpha, 1)
        if normal.ndim != 4 or normal.shape[-1] != 3 or alpha.ndim != 3:
            raise ValueError("video_frames: normal must be [N,H,W,3] and alpha [N,H,W]")
        nrm = frames(out_nrm)
    _lib.launch("srf_video_frames", dev, N, H, W, image.data_ptr(), ctypes.byref(ai), _lib._ptr(normal),
                ctypes.byref(an) if an is not None else None, _lib._ptr(alpha) if normal is not None else 0,
                ctypes.byref(aa) if aa is not None else None, rgb.data_ptr(), _lib._ptr(nrm))
    return rgb, nrm


# forward-only state a chunk of the video may hold on the device; 2 GiB keeps the path's peak memory small next to the
# network's and still renders LaRa's 120 frames of 512^2 with ~0.5 M Gaussians in few chunks
CHUNK_BUDGET_BYTES = 2 << 30


def default_chunk(P: int, H: int, W: int, N: int, device) -> int:
    """Views per chunk: the forward-only rasterizer state of one view (binning at the forward's optimistic capacity) plus
    its epilogue outputs, rays and frames, fitted into :data:`CHUNK_BUDGET_BYTES`."""
    from . import rasterizer as R
    lib = _lib.load()
    state = sum(R._views_sizes(lib, 1, P, H, W, R.initial_capacity(P, device), False)[:5])
    per_view = state + H * W * 4 * (6 + 16) + H * W * 6
    return max(1, min(N, CHUNK_BUDGET_BYTES // max(per_view, 1)))


@torch.no_grad()
def render_video_frames(renderer, gs_params, cams: Sequence, chunk: Optional[int] = None, device="cuda",
                        normals: bool = True):
    """LaRa's video loop (evaluation.py:118-138) in chunks of views: each chunk is rendered forward-only through
    ``renderer.render_views``, quantised on the device by :func:`video_frames` and copied into a pinned host buffer on a
    side stream, so that the copy of one chunk overlaps the render of the next.  ``gs_params`` is LaRa's fine
    ``render_pkg[1]`` (centers, shs, opacity, scaling, rotation, mask).  Returns (rgb, nrm) numpy uint8 [N,H,W,3]
    (nrm None without ``normals``), the frames ``imageio.mimwrite`` takes."""
    centers, shs, opacity, scaling, rotation, mask = gs_params
    opacity, scaling, rotation = opacity[mask], scaling[mask], rotation[mask]
    device = torch.device(device)
    if device.type == "cuda" and device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    N = len(cams)
    if N == 0:
        return np.empty((0, 0, 0, 3), np.uint8), (np.empty((0, 0, 0, 3), np.uint8) if normals else None)
    H, W = int(cams[0].image_height), int(cams[0].image_width)
    if chunk is None:
        chunk = default_chunk(int(centers.shape[0]), H, W, N, device)
    chunk = max(1, min(int(chunk), N))
    host_rgb = torch.empty((N, H, W, 3), dtype=torch.uint8, pin_memory=True)
    host_nrm = torch.empty((N, H, W, 3), dtype=torch.uint8, pin_memory=True) if normals else None
    bufs = [[torch.empty((chunk, H, W, 3), dtype=torch.uint8, device=device) for _ in range(2 if normals else 1)]
            for _ in range(2)]
    copied = [None, None]                      # event: the side stream is done reading bufs[k]
    compute, side = torch.cuda.current_stream(device), torch.cuda.Stream(device)
    for k, a in enumerate(range(0, N, chunk)):
        sub = list(cams[a:a + chunk])
        for cam in sub:
            cam.to_device(device)
        rays = torch.stack([cam.get_rays().squeeze(0) for cam in sub]).to(device)
        out = renderer.render_views(sub, rays, centers, shs, opacity, scaling, rotation, device)
        n, buf = len(sub), bufs[k % 2]
        if copied[k % 2] is not None:
            compute.wait_event(copied[k % 2])
        video_frames(out["image"], out["rend_normal"] if normals else None, out["acc_map"] if normals else None,
                     buf[0][:n], buf[1][:n] if normals else None)
        done = torch.cuda.Event()
        done.record(compute)
        with torch.cuda.stream(side):
            side.wait_event(done)
            host_rgb[a:a + n].copy_(buf[0][:n], non_blocking=True)
            if normals:
                host_nrm[a:a + n].copy_(buf[1][:n], non_blocking=True)
            copied[k % 2] = torch.cuda.Event()
            copied[k % 2].record(side)
            for t in buf:
                t.record_stream(side)
    side.synchronize()
    return host_rgb.numpy(), (host_nrm.numpy() if normals else None)
