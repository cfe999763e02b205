"""Time LaRa's evaluation against the fused path on one GPU (DESIGN §3.22).

* video: LaRa's per-frame loop (evaluation.py:118-136: ``render_img`` per camera, then ``.cpu().numpy()`` and
  ``np.round(x*255).astype('uint8')`` for the RGB and the white-background normal) against
  ``lara_b200.evaluate.render_video_frames`` at its default chunk, 120 frames of 512^2, P Gaussians.
* metrics: ``novel_view_metrics`` against LaRa's torch / NumPy lines (evaluation.py:83-111, tools/depth.py) with a
  plain-torch single-scale SSIM in place of pytorch_msssim, 4 input + 4 novel views of 512^2, four thresholds.

Arms alternate; medians, ranges and peak memory are printed as one JSON line.

    python tools/bench_eval.py [--P 524288] [--frames 120] [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from timing import alternate, card, host_ms, peak_mib, summary  # noqa: E402  (tools/ is on sys.path as a script)


def ssim_torch(X, Y, data_range=1.0):
    """pytorch-msssim 1.0.0 ssim(size_average=False) in plain torch (the library's window and grouped convolutions)."""
    c = torch.arange(11, dtype=torch.float) - 5
    g = torch.exp(-(c ** 2) / (2 * 1.5 ** 2))
    g = (g / g.sum()).to(X)
    C = X.shape[1]
    w = g.reshape(1, 1, 1, 11).repeat(C, 1, 1, 1)
    f = lambda t: F.conv2d(F.conv2d(t, w.transpose(2, 3), groups=C), w, groups=C)      # noqa: E731
    C1, C2 = (0.01 * data_range) ** 2, (0.03 * data_range) ** 2
    mu1, mu2 = f(X), f(Y)
    s1, s2, s12 = f(X * X) - mu1 ** 2, f(Y * Y) - mu2 ** 2, f(X * Y) - mu1 * mu2
    cs = (2 * s12 + C2) / (s1 + s2 + C2)
    return (((2 * mu1 * mu2 + C1) / (mu1 ** 2 + mu2 ** 2 + C1)) * cs).flatten(2).mean(-1).mean(1)


def lara_metrics(out, sample, n_view, thresholds, W):
    images = out["image_fine"][0]
    img_gt = sample["tar_rgb"][0].permute(1, 0, 2, 3).reshape(images.shape)
    images = images.permute(2, 0, 1)[None][..., W * n_view:]
    img_gt = img_gt.permute(2, 0, 1)[None][..., W * n_view:]
    psnr = -10. * torch.log(((images - img_gt) ** 2).mean()) / torch.log(torch.tensor([10.]).to(images.device))
    res = [psnr.item(), ssim_torch(images, img_gt).item()]
    B, N, H, Wd = sample["tar_msk"].shape
    mask = sample["tar_msk"].permute(0, 2, 1, 3).reshape(B, H, N * Wd).cpu().bool().numpy()
    dgt = sample["tar_dep"].permute(0, 2, 1, 3).reshape(B, H, N * Wd).cpu().numpy()
    dp = out["depth_fine"].cpu().squeeze(-1).numpy()
    err = np.abs(dp[mask] - dgt[mask])
    res.append(err.mean().item())
    res += [(err < t).astype("float").mean() for t in thresholds]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=524288)
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_eval needs a GPU"
    from lara_b200 import scene as S
    from lara_b200.evaluate import default_chunk, novel_view_metrics, render_video_frames, video_path
    from lara_b200.renderer import Renderer
    dev = torch.device("cuda:0")
    sc = S.scene(a.P, 0, sh_degree=3)
    params = (sc["means3D"].to(dev), sc["shs"].to(dev), torch.log(sc["opacities"] / (1 - sc["opacities"])).to(dev),
              torch.log(sc["scales"]).to(dev), sc["rotations"].to(dev), torch.ones(a.P, dtype=torch.bool, device=dev))
    renderer = Renderer(sh_degree=3)
    cams = video_path(a.frames, "gobjeverse", (a.size, a.size))
    H = W = a.size

    @torch.no_grad()
    def lara_loop():
        c, s, o, scl, r, m = params
        imgs, nrms = [], []
        for cam in cams:
            cam.to_device(dev)
            rays = cam.get_rays()[0].to(dev)      # this Renderer takes [H,W,6]
            out = renderer.render_img(cam, rays, c, s, o[m], scl[m], r[m], dev)
            img, normal = out["image"], out["rend_normal"]
            imgs.append(np.round(img.cpu().detach().numpy() * 255).astype("uint8"))
            alpha = out["acc_map"][..., None]
            nrms.append(np.round((((normal * alpha + 1 - alpha) + 1) / 2).cpu().detach().numpy() * 255).astype("uint8"))
        return imgs, nrms

    fused = lambda: render_video_frames(renderer, params, cams, device=dev)      # noqa: E731
    lara_loop(), fused()                      # warm-up of every shape
    arms = {"lara_loop": lara_loop, "fused": fused}
    res = alternate(arms, a.reps, host_ms)
    peak = {k: peak_mib(fn) for k, fn in arms.items()}
    r1, n1 = lara_loop()
    r2, n2 = fused()
    same = bool(np.array_equal(np.stack(r1), r2) and np.array_equal(np.stack(n1), n2))

    # metrics at LaRa's eval size: 4 input + 4 novel views
    V, nv, thr = 8, 4, (0.01, 0.02, 0.05, 0.1)
    g = torch.Generator().manual_seed(1)
    tar = torch.rand((1, V, H, W, 3), generator=g)
    img = (tar + 0.05 * torch.randn(tar.shape, generator=g)).clamp(0, 1)
    dgt = torch.rand((1, V, H, W), generator=g) + 1
    dep = dgt + 0.03 * torch.randn(dgt.shape, generator=g)
    msk = (torch.rand((1, V, H, W), generator=g) > 0.4).float()
    out = {"image_fine": img[0].permute(1, 0, 2, 3).reshape(1, H, V * W, 3).to(dev),
           "depth_fine": dep[0].permute(1, 0, 2).reshape(1, H, V * W, 1).to(dev)}
    sample = {"tar_rgb": tar.to(dev), "tar_dep": dgt.to(dev), "tar_msk": msk.to(dev)}
    m_lara = lambda: lara_metrics(out, sample, nv, thr, W)                          # noqa: E731
    m_fused = lambda: novel_view_metrics(out, sample, nv, True, thr)               # noqa: E731
    with torch.no_grad():
        m_lara(), m_fused()
        marms = {"lara_metrics": m_lara, "fused_metrics": m_fused}
        mres = alternate(marms, max(a.reps, 10), host_ms)
        peak.update({k: peak_mib(fn) for k, fn in marms.items()})
        ml, mf = m_lara(), m_fused()

    print(json.dumps({
        "card": card(), "P": a.P, "frames": a.frames, "size": a.size,
        "chunk": default_chunk(a.P, H, W, a.frames, dev),
        **{k: {"ms": summary(v), "peak_mib": round(peak[k], 1)} for k, v in res.items()}, "frames_identical": same,
        **{k: {"ms": summary(v), "peak_mib": round(peak[k], 1)} for k, v in mres.items()},
        "metrics_lara": ml, "metrics_fused": [mf["psnr"], mf["ssim"]] + mf["depth_acc"],
    }))


if __name__ == "__main__":
    main()
