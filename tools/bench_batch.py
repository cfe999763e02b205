"""Time the transfer of LaRa's training batch against the uint8 batch assembled on the GPU (DESIGN §3.23).

* (a) LaRa's transfer: the collated float32 batch of ``gobjverse`` (tar_rgb, tar_nrm, tar_rays, tar_msk,
  tar_rays_down and the small tensors) at B = 3, N = 8, 512² in pageable host memory, moved with ``.to(device)`` per
  tensor, as Lightning's default transfer does, then synchronised.
* (b) ``lara_b200.batch.assemble_batch`` on the uint8 batch of ``GobjverseViews`` in pinned memory, then synchronised.

Arms alternate.  Also: the bytes each arm moves, computed from the shapes; the kernel's own time from CUDA events and
its achieved bytes/s against the H100 SXM's 3.35 TB/s; the same without normals; and, host only, the CPU time of one
``__getitem__`` of LaRa's float32 sample (``GobjverseViews`` plus LaRa's NumPy expansion lines) against
``GobjverseViews.__getitem__``.  One JSON line.

    python tools/bench_batch.py [--reps 20] [--kernel-iters 50]
"""
from __future__ import annotations

import argparse
import itertools
import json
import os
import random
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from lara_b200 import _lib  # noqa: E402
from lara_b200.batch import GobjverseViews, assemble_batch  # noqa: E402
from timing import alternate, card, cuda_ms, host_ms, summary  # noqa: E402  (tools/ is on sys.path as a script)

PEAK_BYTES_PER_S = 3.35e12     # H100 SXM HBM3, data sheet


class Cfg:
    def __init__(self, H, W, load_normal):
        self.data_root, self.split, self.img_size = "synthetic.h5", "train", [H, W]
        self.n_scenes, self.n_group, self.load_normal = 3000000, 4, load_normal


def synthetic_metas(seed, H, W, n_scenes, n_views=12):
    """gobjaverse.h5's keys with seeded contents: cameras at radius 1.5-2.5, uint8 RGBA (alpha 0, 255 or between)."""
    rng = np.random.default_rng(seed)
    metas = {}
    for s in range(n_scenes):
        perm = rng.permutation(n_views)
        scene = {"groups": {f"groups_4_{i}": perm[i::4].copy() for i in range(4)}}
        for v in range(n_views):
            q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
            c2w = np.eye(4, dtype=np.float32)
            c2w[:3, :3] = q
            d = rng.standard_normal(3)
            c2w[:3, 3] = d / np.linalg.norm(d) * rng.uniform(1.5, 2.5)
            img = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
            img[..., 3] = np.where(img[..., 3] < 96, 0, np.where(img[..., 3] > 160, 255, img[..., 3]))
            scene.update({f"c2w_{v}": c2w, f"fov_{v}": rng.uniform(0.4, 0.9, 2).astype(np.float32),
                          f"image_{v}": img, f"normal_{v}": rng.integers(0, 256, (H, W, 3), dtype=np.uint8)})
        metas[f"scene_{s:03d}"] = scene
    return metas


def lara_float_sample(ds, index):
    """LaRa's float32 sample: GobjverseViews' cameras and views, expanded by LaRa's NumPy lines (gobjverse.py:129-138,
    83-84, utils.py:21-34).  Host only; it stands for the per-sample work LaRa's workers do."""
    s = ds[index]
    H, W = (int(v) for v in ds.img_size)
    img = s["tar_rgba"].astype(np.float32) / 255.
    rgb = (img[..., :3] * img[..., -1:] + s["bg_color"][:, None, None, :] * (1 - img[..., -1:])).astype(np.float32)
    msk = (s["tar_rgba"][..., -1] > 0).astype("uint8")
    out = {k: v for k, v in s.items() if k not in ("tar_rgba", "tar_nrm_u8", "i2w", "i2w_down")}
    out.update(tar_rgb=rgb, tar_msk=msk)
    if "tar_nrm_u8" in s:
        n = s["tar_nrm_u8"].astype(np.float32) / 255. * 2 - 1.0
        n = n @ s["transform_mats"][0, :3, :3].T
        out["tar_nrm"] = n.transpose(1, 0, 2, 3).reshape(H, n.shape[0] * W, 3)
    for key, m, h, w in (("tar_rays", s["i2w"], H, W), ("tar_rays_down", s["i2w_down"], H // 16, W // 16)):
        X, Y = np.meshgrid(np.arange(w), np.arange(h))
        XYZ = np.concatenate((X[:, :, None] + 0.5, Y[:, :, None] + 0.5, np.ones_like(X[:, :, None])), axis=-1)
        d = np.stack([XYZ @ mi for mi in m])
        o = np.broadcast_to(s["tar_c2w"][:, None, None, :3, 3], d.shape)
        out[key] = np.concatenate((o, d), axis=-1).astype(np.float32)
    return out


def nbytes(batch):
    return sum(v.numel() * v.element_size() for v in batch.values() if isinstance(v, torch.Tensor))


def kernel_time(raw_dev, dev, iters):
    """ms per srf_batch_assemble launch (CUDA events over ``iters`` launches) and the bytes it moves."""
    out = assemble_batch(raw_dev, dev)
    rgba, nrm = raw_dev["tar_rgba"], raw_dev.get("tar_nrm_u8")
    B, N, H, W = rgba.shape[:4]
    small = [raw_dev[k].contiguous() for k in ("bg_color", "i2w", "i2w_down")]
    origin = raw_dev["tar_c2w"][..., :3, 3].contiguous()
    rot = None if nrm is None else raw_dev["transform_mats"][:, 0, :3, :3].contiguous()
    args = (B, N, H, W, rgba.data_ptr(), _lib._ptr(nrm), small[0].data_ptr(), small[1].data_ptr(), small[2].data_ptr(),
            origin.data_ptr(), _lib._ptr(rot), out["tar_rgb"].data_ptr(), out["tar_msk"].data_ptr(),
            _lib._ptr(out.get("tar_nrm")), out["tar_rays"].data_ptr(), out["tar_rays_down"].data_ptr())
    launch = lambda: _lib.launch("srf_batch_assemble", dev, *args)      # noqa: E731
    for _ in range(5):
        launch()
    ms = cuda_ms(launch, iters)
    written = sum(out[k].numel() * out[k].element_size()
                  for k in ("tar_rgb", "tar_msk", "tar_nrm", "tar_rays", "tar_rays_down") if k in out)
    read = rgba.numel() + (0 if nrm is None else nrm.numel())
    moved = written + read
    return {"ms": round(ms, 4), "bytes_written": written, "bytes_read": read,
            "TB_per_s": round(moved / ms / 1e9, 3), "share_of_3.35TB_per_s": round(moved / ms / 1e9 / 3.35, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=3)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--kernel-iters", type=int, default=50)
    ap.add_argument("--host-reps", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_batch.py needs a GPU"
    dev = torch.device("cuda:0")
    res = {"card": card(), "B": a.B, "N": 8, "H": a.size, "W": a.size}
    metas = synthetic_metas(0, a.size, a.size, a.B + 1)

    for normals in (True, False):
        ds = GobjverseViews(Cfg(a.size, a.size, normals), metas=metas)
        random.seed(0)
        torch.manual_seed(0)
        samples = [ds[i] for i in range(a.B)]
        raw = torch.utils.data.default_collate(samples)
        raw_pinned = {k: (v.pin_memory() if isinstance(v, torch.Tensor) else v) for k, v in raw.items()}
        # arm (a)'s batch: LaRa's float32 tensors, pageable, with the same values
        lara = {k: v.cpu() if isinstance(v, torch.Tensor) else v for k, v in assemble_batch(raw, dev).items()}
        lara = {k: v for k, v in lara.items() if k not in ("i2w", "i2w_down")}
        tag = "normals" if normals else "no_normals"
        arms = {"ms_a_lara_transfer": lambda: [v.to(dev) for v in lara.values() if isinstance(v, torch.Tensor)],
                "ms_b_assemble_batch": lambda: assemble_batch(raw_pinned, dev)}
        alternate(arms, 3, host_ms)          # warm-up of both arms
        times = alternate(arms, a.reps, host_ms)
        raw_dev = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in raw.items()}
        res[tag] = {
            "bytes_a_lara_pageable_float32": nbytes(lara),
            "bytes_b_uint8_pinned": nbytes(raw),
            **{k: summary(v) for k, v in times.items()},
            "kernel": kernel_time(raw_dev, dev, a.kernel_iters),
        }
        if normals:
            ia, ib = itertools.cycle(range(a.B)), itertools.cycle(range(a.B))      # sample r % B in repeat r
            host = alternate({"lara_float32_restatement": lambda: lara_float_sample(ds, next(ia)),
                              "GobjverseViews": lambda: ds[next(ib)]}, a.host_reps, host_ms)
            res["host_only_getitem_ms"] = {k: summary(v) for k, v in host.items()}
        del raw_pinned, raw_dev, lara
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
