"""LaRa's training loss for every scene of a batch at once (``lara_b200.loss.Losses``, DESIGN §3.27), on the GPU.

* Loss, stats and every gradient map against ``batch_losses64`` (test_batch_loss.py) in float64: the kernels' error
  at most twice that of the same restatement run in fp32; ``psnr`` is LaRa's fp32 expression on the float64 mean.
  At LaRa's size (B = 3, 8 target views of 512^2) and at small ragged sizes (H = 161, the smallest MS-SSIM side; W not
  a multiple of 32), with and without the fine pass, iter 1000 / 1001, B = 1.
* Against the recipe it replaces, ``scene_loss(..., ms_ssim=True)`` per scene and pass, through
  ``render_batch_views`` / ``render_batch_subset_views``: per-plane MS-SSIM values and the elementwise gradient maps
  bit for bit, the rest within a stated bound, and the Gaussians' leaf gradients.
* The NULL-fine case of the new entries gives the bits of the one-pass entries; each pass of the two-source MS-SSIM
  gives, plane by plane, the bits of the one-source call on that pass.
* No host synchronisation in the forward and backward; two runs under ``torch.use_deterministic_algorithms(True)`` give
  identical bits; ``no_grad`` works."""
import ctypes

import pytest
import torch

from lara_b200 import _lib
from lara_b200.loss import Losses, scene_loss
from test_batch_loss import batch_losses64, make_outputs

pytestmark = pytest.mark.gpu

GRAD_KEYS = ("image", "image_fine", "rend_normal", "depth_normal", "rend_dist")

CASES = {
    # name: (B, V, H, W, fine, iter)
    "lara_b3_v8_512": (3, 8, 512, 512, True, 5000),
    "ragged_h161_w83": (2, 2, 161, 83, True, 1001),
    "ragged_iter1000": (2, 2, 161, 83, True, 1000),
    "ragged_no_fine": (2, 3, 161, 67, False, 5000),
    "b1": (1, 2, 176, 97, True, 5000),
}


def _leaves(out, dev):
    """fp32 planar leaves on ``dev`` (the batch renders' buffers) and the [B,V,H,W,C] views of them Losses reads."""
    leaves, views = {}, {}
    for k, t in out.items():
        t = t.float().to(dev)
        if t.ndim == 5:
            p = t.permute(0, 1, 4, 2, 3).contiguous().requires_grad_(k in GRAD_KEYS)
            leaves[k], views[k] = p, p.permute(0, 1, 3, 4, 2)
        else:
            p = t.contiguous().requires_grad_(k in GRAD_KEYS)
            leaves[k], views[k] = p, p
    return leaves, views


def _run_fused(out, tar, it, dev):
    leaves, views = _leaves(out, dev)
    loss, stats = Losses()({"tar_rgb": tar.float().to(dev)}, views, it)
    loss.backward()
    grads = {k: leaves[k].grad for k in GRAD_KEYS if k in leaves}
    # planar grads back to the [B,V,H,W,C] layout of the restatement's inputs
    grads = {k: (g.permute(0, 1, 3, 4, 2) if g is not None and g.ndim == 5 else g) for k, g in grads.items()}
    return loss.detach(), stats, grads


def _run_statement(out, tar, it, dev, dtype):
    x = {k: v.float().to(dev).to(dtype).requires_grad_(k in GRAD_KEYS) for k, v in out.items()}
    loss, stats, _ = batch_losses64(tar.float().to(dev).to(dtype), x, it)
    loss.backward()
    return loss.detach(), stats, {k: x[k].grad for k in GRAD_KEYS if k in x}


def _gerr(g, g64):
    if g64 is None:
        return 0.0 if g is None else float(g.abs().max())
    return float((g.double() - g64).abs().max()) / max(float(g64.abs().max()), 1e-300)


@pytest.mark.parametrize("case", list(CASES))
def test_loss_stats_and_gradients_against_float64(cuda_device, case):
    B, V, H, W, fine, it = CASES[case]
    dev = cuda_device
    out, tar = make_outputs(B, V, H, W, 31, fine=fine)
    l64, s64, g64 = _run_statement(out, tar, it, dev, torch.float64)
    l32, s32, g32 = _run_statement(out, tar, it, dev, torch.float32)
    lk, sk, gk = _run_fused(out, tar, it, dev)
    assert list(sk) == list(s64)
    assert ("distortion" in sk) == (it > 1000) and ("mse_fine" in sk) == fine
    e32, ek = abs(float(l32) - float(l64)), abs(float(lk) - float(l64))
    print(f"\n{case}: loss {float(l64):.6f} err fp32 statement {e32:.2e} fused {ek:.2e}")
    assert lk.dtype == torch.float32 and lk.shape == ()
    assert ek <= 2 * e32 + 2 * torch.finfo(torch.float32).eps * abs(float(l64))
    for k in s64:
        a, b, r = sk[k], s32[k], s64[k]
        assert not a.requires_grad and a.is_cuda and a.dtype == torch.float32 and a.shape == r.shape, k
        if k.startswith("psnr"):     # LaRa's fp32 expression on the float64 mean
            mse = s64["mse" + k[4:]].float()
            ref = -10.0 * torch.log(mse) / torch.log(torch.tensor([10.0], device=dev))
            assert float((a - ref).abs().max()) <= 4 * torch.finfo(torch.float32).eps * float(ref.abs().max()), k
            continue
        e32, ek = float((b.double() - r).abs().max()), float((a.double() - r).abs().max())
        print(f"  {k}: {float(r):.6e} err fp32 statement {e32:.2e} fused {ek:.2e}")
        assert ek <= 2 * e32 + 2 * torch.finfo(torch.float32).eps * float(r.abs().max()), k
    for k in g64:
        e32, ek = _gerr(g32[k], g64[k]), _gerr(gk[k], g64[k])
        print(f"  d/d{k}: err / max|g64| fp32 statement {e32:.2e} fused {ek:.2e}")
        assert ek <= 2 * e32 + 1e-6 and ek <= 1e-4, k


# ---- the recipe's per-scene loop through the batch renders ------------------------------------------------------------

def _render(params, settings, rays, masks, shs_fine):
    from lara_b200.multiview import render_batch_subset_views, render_batch_views
    leaves = [p.detach().clone().requires_grad_(True) for p in params]
    out_b = render_batch_views(*leaves, settings, rays=rays, raw_activations=True, keep_binning=True)
    B = leaves[0].shape[0]
    sf = torch.cat([shs_fine[b][masks[b]] for b in range(B)]).detach().requires_grad_(True)
    out_f = render_batch_subset_views(out_b["binning"], masks, sf)
    for o in (out_b, out_f):
        for k, t in o.items():
            if isinstance(t, torch.Tensor) and t.requires_grad:
                t.retain_grad()
    return leaves + [sf], out_b, out_f


def _recipe(out_b, out_f, tar, it):
    B = tar.shape[0]
    loss, stats = 0, {}
    for i in range(B):
        for o, prex in ((out_b, ""), (out_f, "_fine")):
            out = {k: v[i] for k, v in o.items() if not k.startswith("binning")}
            loss_i, st = scene_loss(out, tar[i], it, batch_scenes=B, prex=prex, ms_ssim=True)
            loss = loss + loss_i
            for k, v in st.items():
                stats[k] = stats.get(k, 0) + v
    return loss, stats


@pytest.mark.parametrize("it", [1000, 5000])
def test_against_the_per_scene_recipe(cuda_device, it):
    from test_gpu_batch_views import _batch
    dev = cuda_device
    B, V, P = 3, 8, 131072
    params, settings, rays, shs_fine = _batch(B, V, P, 7, dev)
    g = torch.Generator(device="cuda").manual_seed(3)
    masks = torch.rand(B, P, generator=g, device=dev) < 0.6
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        # the target: the coarse render itself, perturbed, so that MS-SSIM is far from 0 and from 1
        with torch.no_grad():
            from lara_b200.multiview import render_batch_views
            img = render_batch_views(*params, settings, rays=rays, raw_activations=True)["image"]
            tar = (0.8 * img + 0.2 * torch.rand(img.shape, generator=g, device=dev)).clamp(0, 1).contiguous()
        leaves_a, ob_a, of_a = _render(params, settings, rays, masks, shs_fine)
        loss_a, st_a = Losses()({"tar_rgb": tar}, {**ob_a, **of_a}, it)
        loss_a.backward()
        leaves_r, ob_r, of_r = _render(params, settings, rays, masks, shs_fine)
        loss_r, st_r = _recipe(ob_r, of_r, tar, it)
        loss_r.backward()
    finally:
        torch.use_deterministic_algorithms(prev)
    # per-plane MS-SSIM values: the fused call's workspace against each scene's one-source call, bit for bit
    from lara_b200.ssim import _addr, ssim_launch
    lib = _lib.load()
    H, W = tar.shape[2:4]
    lay2 = _lib.ms_ssim_layout(lib, 2 * B, 3, H, V * W)
    x = ob_a["image"].detach().permute(0, 1, 4, 2, 3)
    xf = of_a["image_fine"].detach().permute(0, 1, 4, 2, 3)
    ws, outv = _passes_forward(x, xf, tar, dev)
    val2 = ws[lay2["val"]:lay2["val"] + 8 * 6 * B].view(torch.float64).view(2, B, 3)
    lay1 = _lib.ms_ssim_layout(lib, 1, 3, H, V * W)
    for p, img in enumerate((x, xf)):
        for b in range(B):
            t = tar[b].permute(0, 3, 1, 2)
            _, ws1 = ssim_launch(dev, img[b].data_ptr(), _addr(img[b], True), t.data_ptr(), _addr(t, True),
                                 (1, 3, H, V * W), 1.0, True, True, 5)
            val1 = ws1[lay1["val"]:lay1["val"] + 24].view(torch.float64)
            assert torch.equal(val1, val2[p, b]), (p, b)
    assert torch.equal(outv, torch.stack([st_a["ssim"], st_a["ssim_fine"]]))
    # stats: sums of the recipe's shares, a different summation grouping (within a few fp32 roundings)
    for k in st_a:
        if k.startswith("psnr"):
            continue
        r = st_r[k]
        assert abs(float(st_a[k]) - float(r)) <= 1e-5 * abs(float(r)), k
    assert abs(float(loss_a) - float(loss_r)) <= 1e-6 * abs(float(loss_r))
    # gradient maps: the elementwise terms bit for bit; g_image carries the MS-SSIM gradient, whose per-plane
    # coefficient is the recipe's up to its rounding (scale 1/(3B) against 1/3 and upstream -0.5 against -0.5/B)
    exact = ["rend_normal", "depth_normal", "rend_dist"] if it > 1000 else []
    for k in exact:
        assert torch.equal(ob_a[k].grad, ob_r[k].grad), k
    for k in ("depth", "acc_map"):
        assert ob_a[k].grad is None and ob_r[k].grad is None
    for o_a, o_r, k in ((ob_a, ob_r, "image"), (of_a, of_r, "image_fine")):
        ga, gr = o_a[k].grad, o_r[k].grad
        err = float((ga - gr).abs().max()) / float(gr.abs().max())
        print(f"\nit {it}: d/d{k} differs from the recipe by {err:.2e} of its maximum")
        assert err <= 1e-5, k
    for i, (la, lr) in enumerate(zip(leaves_a, leaves_r)):
        err = float((la.grad - lr.grad).abs().max()) / float(lr.grad.abs().max())
        print(f"  leaf {i}: gradient differs from the recipe by {err:.2e} of its maximum")
        assert err <= 1e-4, i


def _passes_forward(x, xf, tar, dev):
    """srf_ms_ssim_passes_forward on [B,V,3,H,W] views x (and xf or None) against tar [B,V,H,W,3]: (workspace, out)."""
    from lara_b200.loss import _views_addr
    lib = _lib.load()
    B, V, C, H, W = x.shape
    ws = torch.empty(_lib.ms_ssim_passes_workspace_bytes(lib, B, C, H, V * W, xf is not None), dtype=torch.uint8,
                     device=dev)
    out = torch.empty(1 if xf is None else 2, device=dev)
    ax, ay = _views_addr(x), _views_addr(tar.permute(0, 1, 4, 2, 3))
    _lib.launch("srf_ms_ssim_passes_forward", dev, B, C, H, V * W, x.data_ptr(), 0 if xf is None else xf.data_ptr(),
                ctypes.byref(ax), tar.data_ptr(), ctypes.byref(ay), 1.0, ws.data_ptr(), out.data_ptr())
    return ws, out


def _passes_backward(x, xf, tar, ws, up, dx, dxf, accumulate):
    from lara_b200.loss import _views_addr
    B, V, C, H, W = x.shape
    ax, ay, ag = _views_addr(x), _views_addr(tar.permute(0, 1, 4, 2, 3)), _views_addr(dx)
    _lib.launch("srf_ms_ssim_passes_backward", x.device, B, C, H, V * W, x.data_ptr(),
                0 if xf is None else xf.data_ptr(), ctypes.byref(ax), tar.data_ptr(), ctypes.byref(ay), 1.0,
                ws.data_ptr(), up.data_ptr(), dx.data_ptr(), 0 if dxf is None else dxf.data_ptr(), ctypes.byref(ag),
                accumulate)


@pytest.mark.parametrize("shape", [(3, 8, 512, 512), (2, 2, 161, 83)])
def test_one_pass_entries_keep_their_bits(cuda_device, shape):
    """The NULL-fine loss entries are srf_loss_forward / _backward; each pass of the two-source MS-SSIM is the
    one-source call on that pass, plane by plane (values and coefficients), and so are its gradients."""
    from lara_b200.ssim import ssim_launch
    B, V, H, W = shape
    dev = cuda_device
    out, tar = make_outputs(B, V, H, W, 5, fine=True, dtype=torch.float32)
    p = {k: (v.to(dev).permute(0, 1, 4, 2, 3).contiguous() if v.ndim == 5 else v.to(dev).contiguous())
         for k, v in out.items()}
    tar = tar.to(dev)
    lib = _lib.load()
    n = B * V
    ws = torch.empty(_lib.det_loss_passes_workspace_bytes(lib, n, H, W, True) // 8, dtype=torch.float64, device=dev)
    reg = [p["rend_normal"].data_ptr(), p["depth_normal"].data_ptr(), p["acc_map"].data_ptr()]
    s_old, s_null, s_two, s_fine = (torch.empty(k, dtype=torch.float64, device=dev) for k in (3, 3, 4, 3))
    _lib.launch("srf_loss_forward", dev, n, H, W, 1, p["image"].data_ptr(), tar.data_ptr(), *reg,
                p["rend_dist"].data_ptr(), s_old.data_ptr(), ws.data_ptr())
    _lib.launch("srf_loss_passes_forward", dev, n, H, W, 1, p["image"].data_ptr(), 0, tar.data_ptr(), *reg,
                p["rend_dist"].data_ptr(), s_null.data_ptr(), ws.data_ptr())
    _lib.launch("srf_loss_passes_forward", dev, n, H, W, 1, p["image"].data_ptr(), p["image_fine"].data_ptr(),
                tar.data_ptr(), *reg, p["rend_dist"].data_ptr(), s_two.data_ptr(), ws.data_ptr())
    _lib.launch("srf_loss_forward", dev, n, H, W, 0, p["image_fine"].data_ptr(), tar.data_ptr(), 0, 0, 0, 0,
                s_fine.data_ptr(), ws.data_ptr())
    assert torch.equal(s_old, s_null) and torch.equal(s_two[:3], s_old) and torch.equal(s_two[3], s_fine[0])
    up = torch.tensor([0.7], device=dev)
    w = (1.0 / (3 * n * H * W), 1000.0 / (n * H * W), 0.2 / (n * H * W))
    g = {k: torch.empty_like(p[k]) for k in ("image", "image_fine", "rend_normal", "depth_normal", "rend_dist")}
    g_old = {k: torch.empty_like(p[k]) for k in g}
    _lib.launch("srf_loss_backward", dev, n, H, W, 1, *w, p["image"].data_ptr(), tar.data_ptr(), *reg,
                up.data_ptr(), g_old["image"].data_ptr(), g_old["rend_normal"].data_ptr(),
                g_old["depth_normal"].data_ptr(), g_old["rend_dist"].data_ptr())
    _lib.launch("srf_loss_backward", dev, n, H, W, 0, *w, p["image_fine"].data_ptr(), tar.data_ptr(), 0, 0, 0,
                up.data_ptr(), g_old["image_fine"].data_ptr(), 0, 0, 0)
    _lib.launch("srf_loss_passes_backward", dev, n, H, W, 1, *w, p["image"].data_ptr(), p["image_fine"].data_ptr(),
                tar.data_ptr(), *reg, up.data_ptr(), *(g[k].data_ptr() for k in g))
    for k in g:
        assert torch.equal(g[k], g_old[k]), k
    # MS-SSIM: one source (x_fine NULL) against srf_ms_ssim_forward, two sources against each pass alone
    x, xf = p["image"], p["image_fine"]
    lay1, lay2 = _lib.ms_ssim_layout(lib, B, 3, H, V * W), _lib.ms_ssim_layout(lib, 2 * B, 3, H, V * W)
    from lara_b200.loss import _views_addr
    ay = _views_addr(tar.permute(0, 1, 4, 2, 3))
    ws2, out2 = _passes_forward(x, xf, tar, dev)
    gx2, gxf2 = torch.full_like(x, 0.25), torch.full_like(xf, -0.5)
    up2 = torch.tensor([-0.5, -0.25], device=dev)
    _passes_backward(x, xf, tar, ws2, up2, gx2, gxf2, 1)
    P = 3 * B
    for s, img in enumerate((x, xf)):
        out1, ws1 = ssim_launch(dev, img.data_ptr(), _views_addr(img), tar.data_ptr(), ay, (B, 3, H, V * W), 1.0,
                                True, True, 5)
        ws0, out0 = _passes_forward(img, None, tar, dev)
        assert torch.equal(out0, out1.reshape(1))
        assert torch.equal(out2[s], out1), s
        v1 = ws1[lay1["val"]:lay1["val"] + 8 * P].view(torch.float64)
        v2 = ws2[lay2["val"]:lay2["val"] + 16 * P].view(torch.float64)[s * P:(s + 1) * P]
        c1 = ws1[lay1["coef"]:lay1["coef"] + 4 * 5 * P].view(torch.float32).view(5, P)
        c2 = ws2[lay2["coef"]:lay2["coef"] + 4 * 10 * P].view(torch.float32).view(5, 2 * P)[:, s * P:(s + 1) * P]
        assert torch.equal(v1, v2) and torch.equal(c1, c2), s
        g1, g0 = torch.empty_like(img), torch.empty_like(img)
        _lib.launch("srf_ms_ssim_backward", dev, B, 3, H, V * W, img.data_ptr(), ctypes.byref(_views_addr(img)),
                    tar.data_ptr(), ctypes.byref(ay), 1.0, 1, ws1.data_ptr(), up2[s:s + 1].data_ptr(), g1.data_ptr(),
                    ctypes.byref(_views_addr(g1)))
        _passes_backward(img, None, tar, ws0, up2[s:s + 1].contiguous(), g0, None, 0)
        assert torch.equal(g0, g1), s
        assert torch.equal((gx2, gxf2)[s], g1 + (0.25, -0.5)[s]), s


# ---- execution properties -----------------------------------------------------------------------------------------------

def test_no_host_sync_determinism_and_no_grad(cuda_device):
    B, V, H, W = 3, 8, 512, 512
    dev = cuda_device
    out, tar = make_outputs(B, V, H, W, 9, fine=True, dtype=torch.float32)
    tar = tar.to(dev)
    runs = []
    prev = torch.are_deterministic_algorithms_enabled()
    for det in (False, True, True):
        torch.use_deterministic_algorithms(det)
        try:
            leaves, views = _leaves(out, dev)
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
            try:
                loss, stats = Losses()({"tar_rgb": tar}, views, 5000)
                loss.backward()
            finally:
                torch.cuda.set_sync_debug_mode(0)
        finally:
            torch.use_deterministic_algorithms(prev)
        runs.append((loss.detach(), {k: v.clone() for k, v in stats.items()},
                     {k: leaves[k].grad.clone() for k in GRAD_KEYS}))
    (l1, s1, g1), (l2, s2, g2) = runs[1], runs[2]
    assert torch.equal(l1, l2)
    for k in s1:
        assert torch.equal(s1[k], s2[k]), k
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k
    # the default (atomic) sums differ from the deterministic ones by rounding only; the gradient maps do not depend
    # on the sums
    assert abs(float(runs[0][0]) - float(l1)) <= 1e-6 * abs(float(l1))
    for k in g1:
        assert torch.equal(runs[0][2][k], g1[k]), k
    # validation_step: no_grad gives the same loss and stats and builds no graph
    leaves, views = _leaves(out, dev)
    torch.use_deterministic_algorithms(True)
    try:
        with torch.no_grad():
            loss, stats = Losses()({"tar_rgb": tar}, views, 5000)
    finally:
        torch.use_deterministic_algorithms(prev)
    assert not loss.requires_grad and torch.equal(loss, l1)
    for k in s1:
        assert torch.equal(stats[k], s1[k]), k
