"""LaRa's training loss for every scene of a batch at once (lara_b200.loss.Losses, csrc/loss.cu, csrc/ms_ssim.cu).

* ``batch_losses64`` restates, in plain torch, what the fused path computes on the batch renders' [B,V,H,W,C] outputs:
  one squared-error sum per pass and the regulariser sums over all scenes, the MS-SSIM value of every (scene, pass,
  channel) plane of the views side by side, each pass's mean over its planes, and LaRa's loss assembled from them.  In
  float64 it equals the CPU restatement of LaRa's own ``Losses.forward`` (oracle.torch_restatements.lara_loss_torch,
  pinned to LaRa's module by test_ms_ssim.py) on the concatenated [B,H,V*W,C] layout; test_gpu_batch_loss.py checks
  the kernels against it.
* The argument checks of the new C entries and of ``Losses``, before any launch."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from test_ms_ssim import ms_ssim_torch, smooth_pair


def _cat(t):
    """[B,V,H,W,C] or [B,V,H,W] -> LaRa's [B,H,V*W,C] / [B,H,V*W] (network.py's torch.cat of the views)."""
    B, V, H, W = t.shape[:4]
    return t.transpose(1, 2).reshape((B, H, V * W) + tuple(t.shape[4:]))


def plane_ms_ssim(image, tar):
    """MS-SSIM of every (scene, channel) plane of [B,V,H,W,3] against [B,V,H,W,3], the views side by side: [B,3]."""
    B = image.shape[0]
    x, y = _cat(image).permute(0, 3, 1, 2), _cat(tar).permute(0, 3, 1, 2)
    H, VW = x.shape[2:]
    v = ms_ssim_torch(x.reshape(B * 3, 1, H, VW), y.reshape(B * 3, 1, H, VW), data_range=1.0, size_average=False)
    return v.reshape(B, 3)


def batch_losses64(tar, out, it):
    """(loss, stats, parts) of LaRa's Losses on the batch outputs ``out`` ([B,V,H,W,C] as the batch renders give them)
    and ``tar`` [B,V,H,W,3], computed the way the fused path does, in the inputs' dtype.  ``parts`` holds the sums
    (``sse``, ``dist``, ``nerr``, ``sse_fine``) and the per-plane MS-SSIM values (``planes``, ``planes_fine``)."""
    B, V, H, W = tar.shape[:4]
    npx = B * V * H * W
    fine = "acc_map_fine" in out
    with_reg = "rend_dist" in out and it > 1000
    parts = {"sse": ((out["image"] - tar) ** 2).sum(), "planes": plane_ms_ssim(out["image"], tar)}
    if with_reg:
        parts["dist"] = out["rend_dist"].sum()
        parts["nerr"] = ((1 - (out["rend_normal"] * out["depth_normal"]).sum(-1)) * out["acc_map"].detach()).sum()
    if fine:
        parts["sse_fine"] = ((out["image_fine"] - tar) ** 2).sum()
        parts["planes_fine"] = plane_ms_ssim(out["image_fine"], tar)
    stats = {}
    loss = 0
    for prex in ("", "_fine") if fine else ("",):
        mse = parts[f"sse{prex}"] / (3 * npx)
        ssim = parts[f"planes{prex}"].mean()
        stats[f"mse{prex}"] = mse.detach()
        # LaRa's expression: the float32 log(10) makes the result float32 whatever the dtype of mse
        stats[f"psnr{prex}"] = -10.0 * torch.log(mse.detach()) / torch.log(torch.tensor([10.0], device=mse.device))
        stats[f"ssim{prex}"] = ssim.detach()
        loss = loss + mse + 0.5 * (1 - ssim)
        if with_reg and not prex:
            dist, nerr = parts["dist"] / npx, parts["nerr"] / npx
            stats["distortion"], stats["normal"] = dist.detach(), nerr.detach()
            loss = loss + dist * 1000
            loss = loss + nerr * 0.2
    return loss, stats, parts


def make_outputs(B, V, H, W, seed, fine=True, dtype=torch.float64):
    """Batch-render-like outputs {key: [B,V,H,W,C]} and the target [B,V,H,W,3]: smooth images and perturbed copies
    (so that no MS-SSIM level is relu'd to 0), random regularisers."""
    g = torch.Generator().manual_seed(seed + 1000)
    img, tar = smooth_pair(B * V, 3, H, W, seed, dtype=torch.float64)
    r = lambda *s: torch.rand(s, generator=g, dtype=torch.float64)       # noqa: E731
    out = {"image": img.reshape(B, V, 3, H, W).permute(0, 1, 3, 4, 2),
           "rend_dist": r(B, V, H, W) * 0.01, "acc_map": r(B, V, H, W),
           "rend_normal": F.normalize(r(B, V, H, W, 3) - 0.5, dim=-1),
           "depth_normal": F.normalize(r(B, V, H, W, 3) - 0.5, dim=-1)}
    tar = tar.reshape(B, V, 3, H, W).permute(0, 1, 3, 4, 2).contiguous()
    if fine:
        out["image_fine"] = (0.7 * out["image"] + 0.3 * tar + 0.01 * (r(B, V, H, W, 3) - 0.5))
        out["acc_map_fine"] = r(B, V, H, W)
    return {k: v.to(dtype) for k, v in out.items()}, tar.to(dtype)


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("fine", [False, True])
@pytest.mark.parametrize("it", [1000, 5000])
def test_batch_restatement_matches_lara_losses_restatement(B, fine, it):
    from oracle.torch_restatements import lara_loss_torch
    out, tar = make_outputs(B, 2, 164, 88, 7 + B, fine=fine)
    keys = [k for k in out if k != "acc_map_fine"]
    a = {k: (out[k].clone().requires_grad_(k != "acc_map") if k in keys else out[k]) for k in out}
    b = {k: out[k].clone().requires_grad_(k != "acc_map") for k in keys}
    loss_a, st_a, parts = batch_losses64(tar, a, it)
    loss_a.backward()
    # LaRa's module on its own layout: the coarse keys, then the fine pass's image alone (no regularisers)
    cat = {k: _cat(b[k]) for k in ("image", "rend_dist", "acc_map", "rend_normal", "depth_normal")}
    loss_b, st_b = lara_loss_torch(cat, tar, it, ssim=ms_ssim_torch)
    if fine:
        loss_f, st_f = lara_loss_torch({"image": _cat(b["image_fine"])}, tar, it, ssim=ms_ssim_torch)
        loss_b = loss_b + loss_f
        st_b.update({k + "_fine": v for k, v in st_f.items()})
    loss_b.backward()
    assert float(parts["planes"].detach().min()) > 0.1
    assert sorted(st_a) == sorted(st_b)
    assert list(st_a) == list(st_b)
    assert ("distortion" in st_a) == (it > 1000)
    assert abs(float(loss_a) - float(loss_b)) <= 1e-13 * abs(float(loss_b))
    for k in st_a:
        assert st_a[k].shape == st_b[k].shape, k
        assert float((st_a[k] - st_b[k]).abs().max()) <= 1e-13 * float(st_b[k].abs().max()), k
    for k in keys:
        if k == "acc_map":
            assert a[k].grad is None and b[k].grad is None
            continue
        ga, gb = a[k].grad, b[k].grad
        if gb is None:      # the regularisers' inputs at iter <= 1000
            assert ga is None or float(ga.abs().max()) == 0.0, k
            continue
        assert float((ga - gb).abs().max()) <= 1e-12 * float(gb.abs().max()), k


# ---- argument checks (no GPU) -----------------------------------------------------------------------------------------

def test_loss_passes_entries_reject_bad_arguments_before_any_launch(lib):
    n = ctypes.c_size_t()
    assert lib.srf_loss_passes_deterministic_workspace_bytes(24, 512, 512, 1, ctypes.byref(n)) == 0
    assert n.value == 1024 * 4 * 8
    assert lib.srf_loss_passes_deterministic_workspace_bytes(24, 512, 512, 0, ctypes.byref(n)) == 0
    assert n.value == 1024 * 3 * 8
    assert lib.srf_loss_passes_deterministic_workspace_bytes(0, 512, 512, 1, ctypes.byref(n)) != 0
    assert lib.srf_loss_passes_deterministic_workspace_bytes(1, 8, 8, 1, None) != 0

    def fwd(V=1, H=8, W=8, reg=0, image=256, fine=512, tar=768, rn=None, dn=None, acc=None, dist=None, sums=1024, ws=None):
        return lib.srf_loss_passes_forward(None, V, H, W, reg, image, fine, tar, rn, dn, acc, dist, sums, ws)
    assert fwd(V=0) != 0 and b"srf_loss_passes_forward: bad sizes" in lib.srf_last_error()
    assert fwd(H=-1) != 0 and b"bad sizes" in lib.srf_last_error()
    assert fwd(V=1 << 20, H=1 << 14, W=1 << 14) != 0 and b"exceeds" in lib.srf_last_error()
    assert fwd(image=None) != 0 and b"null pointer" in lib.srf_last_error()
    assert fwd(tar=None) != 0 and b"null pointer" in lib.srf_last_error()
    assert fwd(sums=None) != 0 and b"null pointer" in lib.srf_last_error()
    assert fwd(reg=1) != 0 and b"null regulariser input" in lib.srf_last_error()
    assert fwd(fine=514) != 0 and b"4-byte aligned" in lib.srf_last_error()
    assert fwd(image=258) != 0 and b"4-byte aligned" in lib.srf_last_error()
    assert fwd(sums=1028) != 0 and b"sums must be 8-byte aligned" in lib.srf_last_error()
    assert fwd(ws=1028) != 0 and b"workspace" in lib.srf_last_error()

    def bwd(V=1, H=8, W=8, reg=0, image=256, fine=512, tar=768, up=1280, g=1536, gf=1792, grn=None, gdn=None, gd=None):
        return lib.srf_loss_passes_backward(None, V, H, W, reg, 1.0, 1.0, 1.0, image, fine, tar, None, None, None, up,
                                            g, gf, grn, gdn, gd)
    assert bwd(W=0) != 0 and b"srf_loss_passes_backward: bad sizes" in lib.srf_last_error()
    assert bwd(V=1 << 20, H=1 << 14, W=1 << 14) != 0 and b"exceeds" in lib.srf_last_error()
    assert bwd(g=None) != 0 and b"null pointer" in lib.srf_last_error()
    assert bwd(gf=None) != 0 and b"image_fine and g_image_fine go together" in lib.srf_last_error()
    assert bwd(fine=None) != 0 and b"go together" in lib.srf_last_error()
    assert bwd(reg=1) != 0 and b"null regulariser pointer" in lib.srf_last_error()
    assert bwd(gf=1794) != 0 and b"4-byte aligned" in lib.srf_last_error()
    assert bwd(up=1282) != 0 and b"4-byte aligned" in lib.srf_last_error()


def test_ms_ssim_passes_entries_reject_bad_arguments_before_any_launch(lib):
    from lara_b200 import _lib
    n, m = ctypes.c_size_t(), ctypes.c_size_t()
    assert lib.srf_ms_ssim_passes_workspace_bytes(3, 3, 512, 4096, 1, ctypes.byref(n)) == 0
    assert lib.srf_ms_ssim_workspace_bytes(6, 3, 512, 4096, ctypes.byref(m)) == 0 and n.value == m.value
    assert lib.srf_ms_ssim_passes_workspace_bytes(3, 3, 512, 4096, 0, ctypes.byref(n)) == 0
    assert lib.srf_ms_ssim_workspace_bytes(3, 3, 512, 4096, ctypes.byref(m)) == 0 and n.value == m.value
    assert lib.srf_ms_ssim_passes_workspace_bytes(1, 3, 160, 400, 1, ctypes.byref(n)) != 0
    assert b"larger than 160" in lib.srf_last_error()
    assert lib.srf_ms_ssim_passes_workspace_bytes(20000, 3, 176, 176, 0, ctypes.byref(n)) == 0
    assert lib.srf_ms_ssim_passes_workspace_bytes(20000, 3, 176, 176, 1, ctypes.byref(n)) != 0
    assert b"65535" in lib.srf_last_error()
    assert lib.srf_ms_ssim_passes_workspace_bytes(1, 3, 176, 176, 1, None) != 0
    a = _lib.MsSsimAddr(0, 176 * 176, 176, 1, 0, 176)

    def fwd(B=1, H=176, x=256, xf=512, y=768, ws=1024, out=2048, addr=a):
        return lib.srf_ms_ssim_passes_forward(None, B, 3, H, 176, x, xf, ctypes.byref(addr), y, ctypes.byref(a), 1.0,
                                              ws, out)
    assert fwd(H=150) != 0 and b"srf_ms_ssim_passes_forward" in lib.srf_last_error()
    assert fwd(B=0) != 0 and b"bad sizes" in lib.srf_last_error()
    assert fwd(B=20000) != 0 and b"65535" in lib.srf_last_error()
    assert fwd(x=None) != 0 and b"null x" in lib.srf_last_error()
    assert fwd(y=None) != 0 and b"null y" in lib.srf_last_error()
    assert fwd(x=258) != 0 and b"aligned" in lib.srf_last_error()
    assert fwd(xf=514) != 0 and b"x_fine must be 4-byte aligned" in lib.srf_last_error()
    assert fwd(ws=1028) != 0 and b"workspace" in lib.srf_last_error()
    assert fwd(out=None) != 0 and b"null output" in lib.srf_last_error()
    assert fwd(out=2050) != 0 and b"out must be 4-byte aligned" in lib.srf_last_error()
    assert fwd(addr=_lib.MsSsimAddr(0, 1, 1, 1, 0, 0)) != 0 and b"view width" in lib.srf_last_error()

    def bwd(x=256, xf=512, up=1280, dx=1536, dxf=1792, acc=1):
        return lib.srf_ms_ssim_passes_backward(None, 1, 3, 176, 176, x, xf, ctypes.byref(a), 768, ctypes.byref(a), 1.0,
                                               1024, up, dx, dxf, ctypes.byref(a), acc)
    assert bwd(up=None) != 0 and b"upstream" in lib.srf_last_error()
    assert bwd(up=1282) != 0 and b"upstream must be 4-byte aligned" in lib.srf_last_error()
    assert bwd(dx=None) != 0 and b"null dx" in lib.srf_last_error()
    assert bwd(dxf=None) != 0 and b"x_fine and dx_fine go together" in lib.srf_last_error()
    assert bwd(xf=None) != 0 and b"go together" in lib.srf_last_error()
    assert bwd(dxf=1794) != 0 and b"dx_fine must be 4-byte aligned" in lib.srf_last_error()


def _cpu_case(B=2, V=2, H=176, W=96, fine=True):
    out, tar = make_outputs(B, V, H, W, 3, fine=fine, dtype=torch.float32)
    return {"tar_rgb": tar}, out


@pytest.mark.parametrize("case", ["no_tar", "no_image", "no_image_fine", "no_rend_normal", "no_acc_map"])
def test_losses_rejects_missing_keys(case):
    from lara_b200.loss import Losses
    batch, out = _cpu_case()
    if case == "no_tar":
        batch = {}
    else:
        out.pop(case[3:])
    with pytest.raises(KeyError, match=case[3:]):
        Losses()(batch, out, 5000)
    if case in ("no_rend_normal", "no_acc_map"):     # the regularisers are off at iter <= 1000: no error from them
        with pytest.raises(RuntimeError, match="CUDA"):
            Losses()(batch, out, 1000)


@pytest.mark.parametrize("case", ["image_fine", "rend_dist", "tar_rgb", "views", "small"])
def test_losses_rejects_shapes_that_disagree(case):
    from lara_b200.loss import Losses
    batch, out = _cpu_case()
    if case == "image_fine":
        out["image_fine"] = out["image_fine"][:, :, 1:]
    elif case == "rend_dist":
        out["rend_dist"] = out["rend_dist"][..., None]
    elif case == "tar_rgb":
        batch["tar_rgb"] = batch["tar_rgb"][..., :2]
    elif case == "views":
        out["image"] = out["image"][:, :1]
    else:
        batch, out = _cpu_case(V=1)
    with pytest.raises(ValueError):
        Losses()(batch, out, 5000)


def test_losses_rejects_dtypes_and_a_target_that_requires_grad():
    from lara_b200.loss import Losses
    for key in ("image", "image_fine", "depth_normal", "acc_map", "tar_rgb"):
        batch, out = _cpu_case()
        d = batch if key == "tar_rgb" else out
        d[key] = d[key].double()
        with pytest.raises(TypeError, match=key):
            Losses()(batch, out, 5000)
    batch, out = _cpu_case()
    out["image"] = out["image"].half()
    with pytest.raises(TypeError):
        Losses()(batch, out, 10)
    batch, out = _cpu_case()
    batch["tar_rgb"].requires_grad_(True)
    with pytest.raises(RuntimeError, match="requires grad"):
        Losses()(batch, out, 5000)
    batch, out = _cpu_case()
    with pytest.raises(RuntimeError, match="CUDA"):      # every check above runs before the device check
        Losses()(batch, out, 5000)
