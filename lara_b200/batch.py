"""LaRa's training batch on the GPU (``dataLoader/gobjverse.py:40-141``, ``dataLoader/utils.py:21-34``).

LaRa's ``gobjverse`` dataset expands each view to float32 on the host: the composited image, the decoded and rotated
normals and two ray grids, 12.9 MB per 512² view, all of which then crosses PCIe from pageable memory.  Here the
workers keep the uint8 views and the few small per-view matrices, and one kernel (csrc/batch.cu) writes what LaRa's
``Network.forward`` and ``Losses`` read, in LaRa's collated layouts, on the device:

* :class:`GobjverseViews` -- the dataset: LaRa's split selection, view choice and RNG calls (so the same seeds pick
  the same views and backgrounds), its camera re-expression and ``i2w`` matrices, with uint8 ``tar_rgba`` /
  ``tar_nrm_u8`` in place of the float32 images, normals and rays.
* :func:`assemble_batch` -- the collated raw batch (host, pinned or not, or device) -> ``tar_rgb``, ``tar_msk``,
  ``tar_nrm``, ``tar_rays``, ``tar_rays_down`` on the device plus the small tensors moved.
* :func:`batch_cameras` -- the camera records of the batch's target views from ``tar_c2w`` and ``bg_color``, in one
  launch (DESIGN §3.28).

Rounding follows LaRa's NumPy lines: colour and mask bit for bit, the rays bit for bit wherever their three-term fp64
sum is exact, the normals within a stated bound (DESIGN §3.23).
"""
from __future__ import annotations

import random
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib

DOWN = 16           # tar_rays_down is built at 1/16 of the image size
_RAW = ("tar_rgba", "tar_nrm_u8")


def fov_to_ixt(fov: np.ndarray, img_size: np.ndarray) -> np.ndarray:
    """LaRa's intrinsics from ``(fovx, fovy)`` and ``img_size = [H, W]``, rounded as LaRa rounds them.  LaRa's quirk is
    kept: cx and fx come from ``img_size[0]``, which is H, and cy and fy from W."""
    K = np.eye(3, dtype=np.float32)
    K[0, 2] = img_size[0] / 2
    K[1, 2] = img_size[1] / 2
    f = 0.5 * img_size / np.tan(0.5 * fov)            # fp64 (integer img_size), rounded to fp32 on assignment
    K[0, 0], K[1, 1] = f[0], f[1]
    return K


def image_to_world(c2ws: np.ndarray, ixts: np.ndarray, scale: float) -> np.ndarray:
    """``[N,3,3]`` fp32 ``inv(K)^T c2w[:3,:3]^T`` with ``K[:2]`` scaled by ``scale`` (utils.py:24,29): a ray's direction
    at pixel (x, y) is ``(x + 0.5, y + 0.5, 1) @ i2w``."""
    K = ixts.copy()
    K[:, :2] *= scale
    return np.linalg.inv(K).transpose(0, 2, 1) @ c2ws[:, :3, :3].transpose(0, 2, 1)


def _uint8(a, what: str) -> np.ndarray:
    a = np.asarray(a)
    if a.dtype != np.uint8:
        raise TypeError(f"GobjverseViews: {what} must be uint8, got {a.dtype}")
    return a


class GobjverseViews(torch.utils.data.Dataset):
    """LaRa's ``dataLoader.gobjverse`` with uint8 views: the same constructor arguments (``cfg.data_root``, ``split``,
    ``img_size = [H, W]``, ``n_scenes``, ``n_group``, ``load_normal``), split, view choice and RNG calls
    (``torch.randperm`` and ``random.choices`` per group, ``random.choice([0.0, 0.5, 1.0])`` per extra training view,
    in LaRa's order).

    A sample holds LaRa's ``tar_c2w``, ``tar_w2c``, ``tar_ixt``, ``transform_mats``, ``bg_color``, ``near_far``,
    ``fovx``, ``fovy`` and ``meta``, bit for bit, plus ``tar_rgba`` uint8 ``[N,H,W,4]``, ``tar_nrm_u8`` uint8
    ``[N,H,W,3]`` (with ``load_normal``) and ``i2w`` / ``i2w_down`` fp32 ``[N,3,3]``, the matrices LaRa's
    ``build_rays`` forms at full and 1/16 resolution.  :func:`assemble_batch` turns a collated batch of them into
    LaRa's tensors.

    ``metas`` is the opened h5 file, or any mapping with its keys; by default ``h5py.File(cfg.data_root, 'r')``."""

    def __init__(self, cfg, metas=None):
        super().__init__()
        self.cfg = cfg
        self.split = cfg.split
        self.img_size = np.array(cfg.img_size)
        if metas is None:
            import h5py
            metas = h5py.File(cfg.data_root, "r")
        self.metas = metas
        names = np.array(sorted(metas.keys()))
        if "splits" in names:
            self.scenes_name = metas["splits"]["test"][:].astype(str)     # LaRa reads the test list for every split
        else:
            i_test = np.arange(len(names))[::10][:cfg.n_scenes]
            i_train = np.array([i for i in np.arange(len(names)) if i not in i_test])[:cfg.n_scenes]
            self.scenes_name = names[i_train] if self.split == "train" else names[i_test]
        self.n_group = cfg.n_group

    def __len__(self):
        return len(self.scenes_name)

    def _view_ids(self, groups):
        g = self.n_group
        if self.split == "train" and g > 1:
            src = [random.choices(groups[f"groups_{g}_{i}"])[0] for i in torch.randperm(g).tolist()]
            return src + [random.choices(groups[f"groups_{g}_{i}"])[0] for i in torch.randperm(g).tolist()]
        if g == 1:
            return [groups["groups_4_0"][0]] + [groups[f"groups_4_{i}"][-1] for i in range(4)]
        return [groups[f"groups_{g}_{i}"][0] for i in range(g)] + [groups[f"groups_4_{i}"][-1] for i in range(4)]

    def __getitem__(self, index):
        name = self.scenes_name[index]
        scene = self.metas[name]
        view_id = self._view_ids(scene["groups"])
        H, W = self.img_size
        load_normal = self.cfg.load_normal
        rgba, nrm, bgs, c2ws, w2cs, ixts = [], [], [], [], [], []
        for i, idx in enumerate(view_id):
            bg = np.ones(3).astype(np.float32)
            if self.split == "train" and i >= self.n_group:
                bg = bg * random.choice([0.0, 0.5, 1.0])
            bgs.append(bg)
            img = _uint8(scene[f"image_{idx}"], f"image_{idx}")
            if img.shape != (H, W, 4):
                raise ValueError(f"GobjverseViews: image_{idx} is {img.shape}, expected {(int(H), int(W), 4)}")
            rgba.append(img)
            if load_normal:
                n = _uint8(scene[f"normal_{idx}"], f"normal_{idx}")
                if n.shape != (H, W, 3):
                    raise ValueError(f"GobjverseViews: normal_{idx} is {n.shape}, expected {(int(H), int(W), 3)}")
                nrm.append(n)
            c2w = np.array(scene[f"c2w_{idx}"], dtype=np.float32)
            c2ws.append(c2w)
            w2cs.append(np.linalg.inv(c2w))
            ixts.append(fov_to_ixt(np.array(scene[f"fov_{idx}"], dtype=np.float32), self.img_size))
        c2ws, w2cs, ixts = np.stack(c2ws), np.stack(w2cs), np.stack(ixts)

        # the cameras re-expressed with the first view at (0, 0, -r) (gobjverse.py:58-66)
        r = np.linalg.norm(c2ws[0, :3, 3])
        ref_c2w = np.eye(4, dtype=np.float32).reshape(1, 4, 4)
        ref_w2c = np.eye(4, dtype=np.float32).reshape(1, 4, 4)
        ref_c2w[:, 2, 3], ref_w2c[:, 2, 3] = -r, r
        transform_mats = ref_c2w @ w2cs[:1]
        w2cs = w2cs @ c2ws[:1] @ ref_w2c
        c2ws = transform_mats @ c2ws

        ret = {"fovx": scene["fov_0"][0], "fovy": scene["fov_0"][1],
               "tar_c2w": c2ws, "tar_w2c": w2cs, "tar_ixt": ixts, "transform_mats": transform_mats,
               "bg_color": np.stack(bgs), "tar_rgba": np.stack(rgba)}
        if load_normal:
            ret["tar_nrm_u8"] = np.stack(nrm)
        ret["near_far"] = np.array([r - 0.8, r + 0.8]).astype(np.float32)
        ret["meta"] = {"scene": name, "tar_view": view_id, "frame_id": 0, "tar_h": int(H), "tar_w": int(W)}
        ret["i2w"] = image_to_world(c2ws, ixts, 1.0)
        ret["i2w_down"] = image_to_world(c2ws, ixts, 1.0 / DOWN)
        return ret


def _check_f32(t: torch.Tensor, name: str, shape) -> None:
    if t.dtype != torch.float32:
        raise TypeError(f"assemble_batch: {name} must be float32, got {t.dtype}")
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"assemble_batch: {name} must be {list(shape)}, got {list(t.shape)}")


@torch.no_grad()
def assemble_batch(raw: Dict, device: Optional[torch.device] = None) -> Dict:
    """The dict LaRa's ``Network.forward`` and ``Losses`` read, from a collated batch of :class:`GobjverseViews`
    samples: ``tar_rgb`` f32 ``[B,N,H,W,3]``, ``tar_msk`` u8 ``[B,N,H,W]``, ``tar_nrm`` f32 ``[B,H,N*W,3]`` (when the
    batch has ``tar_nrm_u8``), ``tar_rays`` f32 ``[B,N,H,W,6]`` and ``tar_rays_down`` f32 ``[B,N,H//16,W//16,6]``, on
    ``device``, plus every other tensor of ``raw`` moved there (``meta`` is passed through as it is).

    ``raw`` may be on the host or already on the device (as after Lightning's own transfer).  Host tensors are copied
    with ``non_blocking=True``, which overlaps with the host only from pinned memory (``DataLoader(pin_memory=True)``);
    everything is enqueued on the current stream, and the outputs are fresh tensors.  ``device`` defaults to the batch's
    CUDA device, or the current one for a host batch."""
    rgba = raw["tar_rgba"]
    if rgba.dtype != torch.uint8:
        raise TypeError(f"assemble_batch: tar_rgba must be uint8, got {rgba.dtype}")
    if rgba.ndim != 5 or rgba.shape[-1] != 4:
        raise ValueError(f"assemble_batch: tar_rgba must be [B,N,H,W,4], got {list(rgba.shape)}")
    B, N, H, W = (int(s) for s in rgba.shape[:4])
    if device is None:
        device = rgba.device if rgba.is_cuda else torch.device("cuda", torch.cuda.current_device())
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError(f"assemble_batch: the batch is assembled on a CUDA device, not {dev}")
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())

    nrm = raw.get("tar_nrm_u8")
    if nrm is not None:
        if nrm.dtype != torch.uint8:
            raise TypeError(f"assemble_batch: tar_nrm_u8 must be uint8, got {nrm.dtype}")
        if tuple(nrm.shape) != (B, N, H, W, 3):
            raise ValueError(f"assemble_batch: tar_nrm_u8 must be {[B, N, H, W, 3]}, got {list(nrm.shape)}")
    _check_f32(raw["i2w"], "i2w", (B, N, 3, 3))
    _check_f32(raw["i2w_down"], "i2w_down", (B, N, 3, 3))
    _check_f32(raw["bg_color"], "bg_color", (B, N, 3))
    _check_f32(raw["tar_c2w"], "tar_c2w", (B, N, 4, 4))
    if nrm is not None:
        _check_f32(raw["transform_mats"], "transform_mats", (B, 1, 4, 4))

    def move(t):
        return t.to(dev, non_blocking=True) if isinstance(t, torch.Tensor) else t

    out = {k: move(v) for k, v in raw.items() if k not in _RAW}
    rgba = move(rgba).contiguous()
    nrm = None if nrm is None else move(nrm).contiguous()
    i2w, i2w_down, bg = (out[k].contiguous() for k in ("i2w", "i2w_down", "bg_color"))
    origin = out["tar_c2w"][..., :3, 3].contiguous()
    rot = None if nrm is None else out["transform_mats"][:, 0, :3, :3].contiguous()

    f32 = dict(dtype=torch.float32, device=dev)
    out["tar_rgb"] = torch.empty((B, N, H, W, 3), **f32)
    out["tar_msk"] = torch.empty((B, N, H, W), dtype=torch.uint8, device=dev)
    out["tar_rays"] = torch.empty((B, N, H, W, 6), **f32)
    out["tar_rays_down"] = torch.empty((B, N, H // DOWN, W // DOWN, 6), **f32)
    if nrm is not None:
        out["tar_nrm"] = torch.empty((B, H, N * W, 3), **f32)
    _lib.launch("srf_batch_assemble", dev, B, N, H, W, rgba.data_ptr(), _lib._ptr(nrm), bg.data_ptr(),
                i2w.data_ptr(), i2w_down.data_ptr(), origin.data_ptr(), _lib._ptr(rot), out["tar_rgb"].data_ptr(),
                out["tar_msk"].data_ptr(), _lib._ptr(out.get("tar_nrm")), out["tar_rays"].data_ptr(),
                out["tar_rays_down"].data_ptr())
    return out


def batch_cameras(tar_c2w: torch.Tensor, bg_color: torch.Tensor) -> torch.Tensor:
    """The camera records ``[B*V, SRF_CAM_FLOATS]`` of a batch's target views, built in one launch from the batch's
    ``tar_c2w`` f32 ``[B,V,4,4]`` (or ``[B*V,4,4]``) and ``bg_color`` ``[B,V,3]`` on the device: what
    ``rasterizer.pack_cameras`` builds from LaRa's ``MiniCam`` of each view (lightning/network.py:489-492,
    lightning/utils.py:22-48), with no host read.  The view matrix is ``inverse(c2w)^T`` computed in fp64 and rounded
    once to fp32 (MiniCam's is torch's fp32 inverse), ``campos`` is MiniCam's ``-c2w[:3,3]``.  A pose with a
    non-finite entry or ``|det| < 1e-12`` gets a record that renders the view's background only, where ``MiniCam``'s
    ``torch.inverse`` would raise (include/surfel_batch.h)."""
    fn = "batch_cameras"
    for name, t in (("tar_c2w", tar_c2w), ("bg_color", bg_color)):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{fn}: {name} must be a tensor")
        if t.dtype != torch.float32:
            raise TypeError(f"{fn}: {name} must be float32, got {t.dtype}")
    if tar_c2w.ndim < 3 or tuple(tar_c2w.shape[-2:]) != (4, 4):
        raise ValueError(f"{fn}: tar_c2w must be [B,V,4,4] or [B*V,4,4], got {list(tar_c2w.shape)}")
    n = tar_c2w.numel() // 16
    if bg_color.numel() != 3 * n or bg_color.shape[-1] != 3 or tuple(bg_color.shape[:-1]) != tuple(tar_c2w.shape[:-2]):
        raise ValueError(f"{fn}: bg_color must be {list(tar_c2w.shape[:-2]) + [3]}, got {list(bg_color.shape)}")
    if not 0 < n <= 65535:
        raise ValueError(f"{fn}: {n} views; the records are built for 1 to 65535 views")
    dev = tar_c2w.device
    if dev.type != "cuda" or bg_color.device != dev:
        raise RuntimeError(f"{fn}: tar_c2w and bg_color must be CUDA tensors on one device, got {dev} and "
                           f"{bg_color.device}")
    c2w, bg = tar_c2w.detach().contiguous(), bg_color.detach().contiguous()
    cams = torch.empty((n, _lib.CAM_FLOATS), dtype=torch.float32, device=dev)
    _lib.launch("srf_batch_cameras", dev, n, c2w.data_ptr(), bg.data_ptr(), cams.data_ptr())
    return cams
