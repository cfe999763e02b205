"""LaRa's evaluation on the GPU (lara_b200.ssim.ssim, lara_b200.evaluate) on an H100.

* SSIM value and gradient against the float64 restatement.  Tolerance: the kernels run MS-SSIM's level-0 code, whose
  error bound is checked element by element in test_ms_ssim_per_element; here each case must be within twice the
  error of the same restatement run in fp32 (the library's own precision), and within 5e-6 (value) / 2e-4 (gradient,
  relative to max |g64|) outright.
* Metric counts exact, sums within the fp64 reduction bound, PSNR to 1e-12 of the float64 statement.
* Frames byte for byte against LaRa's recorded expressions, and the chunked video against per-frame renders.
"""
from __future__ import annotations

import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from helpers import reference_record  # noqa: E402
from test_eval import _frame_inputs, frames_chain_np, ssim_pair, ssim_torch  # noqa: E402

pytestmark = pytest.mark.gpu


def _run(fn, x, y, **kw):
    xl = x.detach().clone().requires_grad_(True)
    v = fn(xl, y, **kw)
    v.sum().backward()
    return v.detach().double().cpu(), xl.grad.double().cpu()


SSIM_CASES = {
    # name: (B, C, H, W, seed, data_range, size_average, nonnegative, negative plane, channel-last)
    "odd_2x3x177x211": (2, 3, 177, 211, 21, 1.0, True, False, False, False),
    "H11": (2, 3, 11, 97, 22, 1.0, False, False, False, True),
    "W11": (1, 3, 75, 11, 23, 255.0, True, False, False, False),
    "tile_edges_W64_H32": (2, 3, 32, 64, 24, 1.0, True, False, False, False),
    "tile_edges_W43_H27": (2, 3, 27, 43, 25, 1.0, False, False, False, True),
    "nonnegative_negative_plane": (2, 3, 61, 77, 26, 1.0, False, True, True, False),
}


@pytest.mark.parametrize("case", list(SSIM_CASES))
def test_ssim_against_float64(cuda_device, case):
    from lara_b200.ssim import ssim
    B, C, H, W, seed, R, size_average, nonneg, negative, channel_last = SSIM_CASES[case]
    X64, Y64 = ssim_pair(B, C, H, W, seed, negative)
    X64, Y64 = (X64 * R).to(cuda_device), (Y64 * R).to(cuda_device)
    Xk, Yk = X64.float(), Y64.float()
    if channel_last:
        Xk = Xk.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
        Yk = Yk.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    kw = dict(data_range=R, size_average=size_average, nonnegative_ssim=nonneg)
    X64, Y64 = Xk.double().contiguous(), Yk.double().contiguous()      # float64 on the kernels' own fp32 inputs
    v64, g64 = _run(ssim_torch, X64, Y64, **kw)
    v32, g32 = _run(ssim_torch, Xk.float().contiguous(), Yk.float().contiguous(), **kw)
    vk, gk = _run(ssim, Xk, Yk, **kw)
    gmax = float(g64.abs().max())
    e32 = (float((v32 - v64).abs().max()), float((g32 - g64).abs().max()) / gmax)
    ek = (float((vk - v64).abs().max()), float((gk - g64).abs().max()) / gmax)
    print(f"\n{case}: value {v64.numpy()} errors vs float64 (value abs, grad rel): fp32 restatement {e32}, kernels {ek}")
    assert ek[0] <= 2 * e32[0] + 1e-7 and ek[0] <= 5e-6
    assert ek[1] <= 2 * e32[1] + 1e-6 and ek[1] <= 2e-4
    if nonneg and negative:
        assert float(gk[0, 1].abs().max()) == 0.0


def _lara_views(V, H, W, seed, dev):
    """Planar renders [V,3,H,W] and LaRa's [V,H,W,3] targets (slightly perturbed copies)."""
    X, Y = ssim_pair(V, 3, H, W, seed, False)
    return X.float().to(dev), Y.float().permute(0, 2, 3, 1).contiguous().to(dev)


def test_ssim_views_lara_eval_layout_and_bit_identity(cuda_device):
    """4 novel views of 512^2 side by side: against float64, and bit for bit equal to the contiguous concatenation."""
    from lara_b200.ssim import ssim, ssim_views
    img, tar = _lara_views(8, 512, 512, 31, cuda_device)
    tgt = tar.permute(0, 3, 1, 2)
    vk, gk = _run(lambda x, y: ssim_views(x, y, 1.0, view_range=(4, 8)), img, tgt)
    cat = lambda t: torch.cat(list(t[4:]), dim=-1).unsqueeze(0)        # noqa: E731
    v64, g64 = _run(lambda x, y: ssim_torch(cat(x), cat(y), 1.0, False), img.double(), tgt.double())
    v32, _ = _run(lambda x, y: ssim_torch(cat(x), cat(y), 1.0, False), img, tgt.contiguous())
    gmax = float(g64.abs().max())
    assert abs(float(vk) - float(v64)) <= 2 * abs(float(v32) - float(v64)) + 1e-7
    assert float((gk - g64).abs().max()) / gmax <= 1e-4
    assert float(gk[:4].abs().max()) == 0.0
    vc, gc = _run(lambda x, y: ssim(x, y, 1.0, size_average=True), cat(img).contiguous(), cat(tgt).contiguous())
    assert torch.equal(vk, vc)
    assert torch.equal(gk[4:], torch.stack(gc[0].split(512, dim=-1)))


def test_ssim_repeats_and_deterministic_mode_are_bit_identical(cuda_device):
    from lara_b200.ssim import ssim
    X, Y = (t.float().to(cuda_device) for t in ssim_pair(3, 3, 130, 150, 41, False))
    ref = _run(ssim, X, Y, data_range=1.0, size_average=False)
    assert all(torch.equal(a, b) for a, b in zip(ref, _run(ssim, X, Y, data_range=1.0, size_average=False)))
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        det = _run(ssim, X, Y, data_range=1.0, size_average=False)
    finally:
        torch.use_deterministic_algorithms(prev)
    assert all(torch.equal(a, b) for a, b in zip(ref, det))


# ---- metrics ----

def _metric_scene(V, H, W, seed, dev, empty_mask=False):
    g = torch.Generator().manual_seed(seed)
    tar = torch.rand((1, V, H, W, 3), generator=g)
    img = (tar + 0.05 * torch.randn((1, V, H, W, 3), generator=g)).clamp(0, 1)
    dgt = torch.rand((1, V, H, W), generator=g) * 2 + 0.5
    dep = dgt + 0.05 * torch.randn((1, V, H, W), generator=g)
    msk = (torch.rand((1, V, H, W), generator=g) > 0.3).float()
    if empty_mask:
        msk.zero_()
    # errors exactly fp32(0.01), which lies below 0.01 (not < 0.01 in fp32, < 0.01 in double), and fp32(0.05)
    dgt.view(-1)[:200] = 0.0
    dep.view(-1)[:100] = float(np.float32(0.01))
    dep.view(-1)[100:200] = float(np.float32(0.05))
    msk.view(-1)[:200] = 0.0 if empty_mask else 1.0
    lara_out = {"image_fine": img[0].permute(1, 0, 2, 3).reshape(1, H, V * W, 3),
                "depth_fine": dep[0].permute(1, 0, 2).reshape(1, H, V * W, 1)}
    sample = {"tar_rgb": tar, "tar_dep": dgt, "tar_msk": msk}
    to = lambda d: {k: v.to(dev) for k, v in d.items()}               # noqa: E731
    return to(lara_out), to(sample), img[0], dep[0]


def _numpy_metrics(lara_out, sample, n_views, thresholds, only_novel=True):
    """evaluation.py:83-111 and tools/depth.py, restated on host copies: float64 PSNR, LaRa's fp32 torch PSNR, and the
    depth numbers with NumPy's own comparison of the float32 errors with Python floats."""
    V, H, W = sample["tar_rgb"].shape[1:4]
    images = lara_out["image_fine"][0].cpu()
    img_gt = sample["tar_rgb"][0].cpu().permute(1, 0, 2, 3).reshape(images.shape)
    x0 = W * n_views if only_novel else 0
    images, img_gt = images.permute(2, 0, 1)[None][..., x0:], img_gt.permute(2, 0, 1)[None][..., x0:]
    res = {}
    if images.shape[-1] > 0:
        res["psnr64"] = -10 * math.log10(float(((images - img_gt) ** 2).double().mean()))
        cl = (images - img_gt) ** 2
        res["psnr32"] = float(-10. * torch.log(cl.mean()) / torch.log(torch.tensor([10.])))
    mask = sample["tar_msk"].cpu().permute(0, 2, 1, 3).reshape(1, H, V * W).bool().numpy()
    dgt = sample["tar_dep"].cpu().permute(0, 2, 1, 3).reshape(1, H, V * W).numpy()
    dp = lara_out["depth_fine"].cpu().squeeze(-1).numpy()
    err = np.abs(dp[mask] - dgt[mask])
    res["abs_sum64"] = float(err.astype(np.float64).sum())
    res["count"] = int(mask.sum())
    res["acc_counts"] = [int((err < t).sum()) for t in thresholds]
    return res


THRESHOLDS = (0.01, 0.05, 0.1, 0.2)


@pytest.mark.parametrize("layout", ["lara", "planar", "per_view"])
def test_metrics_against_numpy(cuda_device, layout):
    from lara_b200.evaluate import novel_view_metrics
    V, H, W, nv = 6, 96, 80, 2
    lara_out, sample, img, dep = _metric_scene(V, H, W, 51, cuda_device)
    out = lara_out
    if layout == "planar":
        out = {"image_fine": img.permute(0, 3, 1, 2).contiguous().to(cuda_device), "depth_fine": dep.to(cuda_device)}
    elif layout == "per_view":
        out = {"image_fine": img.to(cuda_device), "depth_fine": dep[..., None].to(cuda_device)}
    m = novel_view_metrics(out, sample, nv, True, THRESHOLDS)
    ref = _numpy_metrics(lara_out, sample, nv, THRESHOLDS)
    assert ref["acc_counts"][0] < ref["acc_counts"][1]
    assert abs(m["psnr"] - ref["psnr64"]) <= 1e-12 * abs(ref["psnr64"])
    assert abs(m["psnr"] - ref["psnr32"]) <= 1e-5 * abs(ref["psnr32"])
    assert abs(m["depth_acc"][0] * ref["count"] - ref["abs_sum64"]) <= 1e-12 * ref["abs_sum64"]
    assert [round(a * ref["count"]) for a in m["depth_acc"][1:]] == ref["acc_counts"]
    assert m["depth_acc"][1:] == [c / ref["count"] for c in ref["acc_counts"]]
    # the errors at exactly fp32(0.01) are not < 0.01 for NumPy: the fp32 comparison
    assert ref["acc_counts"][0] == int(((np.abs(dep.numpy() - sample["tar_dep"][0].cpu().numpy()) <
                                         np.float32(0.01)) & (sample["tar_msk"][0].cpu().numpy() != 0)).sum())
    from lara_b200.ssim import ssim_views
    s = ssim_views(img.permute(0, 3, 1, 2).contiguous().to(cuda_device), sample["tar_rgb"][0].permute(0, 3, 1, 2),
                   1.0, view_range=(nv, V))
    assert m["ssim"] == float(s)


def test_metrics_empty_mask_and_zero_width_range(cuda_device):
    from lara_b200.evaluate import novel_view_metrics
    V, H, W = 3, 32, 24
    lara_out, sample, _, _ = _metric_scene(V, H, W, 52, cuda_device, empty_mask=True)
    m = novel_view_metrics(lara_out, sample, V, True, THRESHOLDS)
    assert m["psnr"] is None and m["ssim"] is None
    assert len(m["depth_acc"]) == 1 + len(THRESHOLDS) and all(math.isnan(v) for v in m["depth_acc"])
    m = novel_view_metrics(lara_out, sample, 1, False, ())
    ref = _numpy_metrics(lara_out, sample, 1, (), only_novel=False)
    assert abs(m["psnr"] - ref["psnr64"]) <= 1e-12 * abs(ref["psnr64"]) and "depth_acc" not in m


def test_metrics_repeat_bit_identical(cuda_device):
    from lara_b200.evaluate import novel_view_metrics
    lara_out, sample, _, _ = _metric_scene(4, 64, 64, 53, cuda_device)
    a = novel_view_metrics(lara_out, sample, 1, True, THRESHOLDS)
    assert a == novel_view_metrics(lara_out, sample, 1, True, THRESHOLDS)


# ---- frames ----

def test_frames_equal_lara_record(cuda_device):
    from lara_b200.evaluate import video_frames
    rec = reference_record("test_eval", "frames")
    img, normal, alpha = _frame_inputs()
    rgb, nrm = video_frames(img.to(cuda_device), normal.to(cuda_device), alpha.to(cuda_device))
    rgb, nrm = rgb.cpu().numpy(), nrm.cpu().numpy()
    inside = (img.numpy() >= 0) & (img.numpy() <= 1)
    assert np.array_equal(rgb[inside], rec["rgb"][inside])
    assert np.array_equal(nrm, rec["nrm"])
    # outside [0, 1]: saturation
    x = img.numpy()
    assert (rgb[x < 0] == 0).all() and (rgb[x > 1] == 255).all()
    # strided inputs (planar storage read channel-last) give the same bytes
    rgb2, nrm2 = video_frames(img.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1).to(cuda_device),
                              normal.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1).to(cuda_device),
                              alpha.to(cuda_device))
    assert np.array_equal(rgb2.cpu().numpy(), rgb) and np.array_equal(nrm2.cpu().numpy(), nrm)


def _video_scene(P, dev, seed=0):
    from lara_b200 import scene as S
    sc = S.scene(P, seed, sh_degree=1)
    logit = lambda p: torch.log(p / (1 - p))          # noqa: E731
    mask = torch.ones(P, dtype=torch.bool)
    return (sc["means3D"].to(dev), sc["shs"].to(dev), logit(sc["opacities"]).to(dev),
            torch.log(sc["scales"]).to(dev), sc["rotations"].to(dev), mask.to(dev))


@pytest.mark.parametrize("P", [60000, 0])
def test_render_video_frames_equal_per_frame_renders(cuda_device, P):
    from lara_b200.evaluate import render_video_frames, video_path
    from lara_b200.renderer import Renderer
    renderer = Renderer(sh_degree=1)
    params = _video_scene(P, cuda_device)
    N, H, W = 120, 128, 128
    cams = video_path(N, "gobjeverse", (W, H))
    with torch.no_grad():
        ref_rgb, ref_nrm = [], []
        c, s, o, sc, r, m = params
        for cam in cams:
            cam.to_device(cuda_device)
            out = renderer.render_img(cam, cam.get_rays()[0].to(cuda_device), c, s, o[m], sc[m], r[m], cuda_device)
            rgb, nrm = frames_chain_np(out["image"].cpu().numpy(), out["rend_normal"].cpu().numpy(),
                                       out["acc_map"].cpu().numpy())
            ref_rgb.append(rgb)
            ref_nrm.append(nrm)
    ref_rgb, ref_nrm = np.stack(ref_rgb), np.stack(ref_nrm)
    if P:
        assert ref_rgb.std() > 1.0
    for chunk in (1, 7, N):
        rgb, nrm = render_video_frames(renderer, params, cams, chunk=chunk, device=cuda_device)
        assert rgb.shape == (N, H, W, 3) and rgb.dtype == np.uint8
        assert np.array_equal(rgb, ref_rgb), chunk
        assert np.array_equal(nrm, ref_nrm), chunk
