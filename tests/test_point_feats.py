"""Fine-pass point-feature sampler (Network.get_point_feats, lightning/network.py:390-411, projection :182-187).

* CPU: the torch restatement ``point_feats_torch`` (below) is pinned bit for bit against LaRa's own ``get_point_feats``
  + ``projection``, forward and autograd gradients under a seeded upstream gradient; LaRa's outputs are recorded in
  tests/golden/reference/test_point_feats.npz by record_reference:

      python tests/test_point_feats.py OUT_DIR LARA_CHECKOUT && cp OUT_DIR/test_point_feats.npz tests/golden/reference/

  The argument checks of the Python entry and of the C entries run without a GPU.
* GPU: the fused kernels vs the restatement (features and rendering gradients to 1e-5 of their maximum, point
  gradients to 1e-4 away from the pixel-centre lines where they jump), the z = 0 case, and an end-to-end check that
  the sampler's gradient reaches the rasterizer's parameters through the permuted views of render_scene_views.
"""
import ctypes
import os
import sys
import types

import numpy as np
import pytest
import torch

from helpers import fingerprint, reference_record, rel_err
from test_decoder_layout import _import_reference_network

FOV = 0.75


def point_feats_torch(points, img_ref, renderings, src_w2cs, src_ixts):
    """Plain-torch restatement of Network.get_point_feats (lightning/network.py:390-411) after the mask gather
    (``points`` is ``points[mask]``), with ``projection`` (:182-187) inlined: what LaRa executes today, and the checker
    of the fused kernels.  src_w2cs [V,4,4], src_ixts [V,3,3]; renderings: image [V,H,W,3], acc_map [V,H,W],
    depth [V,H,W,1].  Returns the [V,8,n] features."""
    n_views_sel, n_points = src_w2cs.shape[0], points.shape[0]
    h, w = img_ref.shape[-2:]
    img_wh = torch.tensor([w, h], device=points.device)
    cam = points.reshape(1, -1, 3) @ src_w2cs[:, :3, :3].permute(0, 2, 1) + src_w2cs[:, :3, 3][:, None]
    cam = cam @ src_ixts.permute(0, 2, 1)
    point_xy, point_z = cam[..., :2] / cam[..., -1:], cam[..., -1:]
    point_xy = (point_xy + 0.5) / img_wh * 2 - 1.0
    stack = torch.cat((renderings["image"], renderings["acc_map"].unsqueeze(-1), renderings["depth"]), dim=-1)
    stack = torch.cat((img_ref, torch.einsum("bhwc->bchw", stack)), dim=1)
    feats = torch.nn.functional.grid_sample(stack, point_xy.unsqueeze(1), align_corners=False)
    feats = feats.view(n_views_sel, -1, n_points).to(stack)
    z_diff = (feats[:, -1:] - point_z.view(n_views_sel, -1, n_points)).abs()
    return torch.cat((feats[:, :-1], z_diff), dim=1)


def lara_cameras(V, H, W, seed=0):
    """(cameras, w2c [V,4,4], ixt [V,3,3]) for V cameras of lara_b200.scene.cameras, with the matrices LaRa's loader
    hands to get_point_feats: w2c = viewmatrix^T, and the pinhole intrinsics of dataLoader/gobjverse.py:10-15
    (focal 0.5*size/tan(fov/2), principal point at the image centre)."""
    from lara_b200 import scene as S
    cams = S.cameras(V, H, W, seed, fov=FOV)
    w2c = torch.stack([c.viewmatrix.T for c in cams]).contiguous()
    size = np.array([W, H])
    focal = 0.5 * size / np.tan(0.5 * FOV)
    ixt = np.eye(3, dtype=np.float32)
    ixt[0, 0], ixt[1, 1], ixt[0, 2], ixt[1, 2] = focal[0], focal[1], W / 2, H / 2
    return cams, w2c, torch.from_numpy(np.stack([ixt] * V))


def _field(g, shape, H, W, coarse):
    """Seeded random images; coarse > 1 gives smooth ones (noise on a grid `coarse` times coarser, upsampled)."""
    if coarse <= 1:
        return torch.rand(shape, generator=g)
    lead = shape[:-2]
    low = torch.rand((int(np.prod(lead)), 1, -(-H // coarse) + 1, -(-W // coarse) + 1), generator=g)
    up = torch.nn.functional.interpolate(low, size=(H, W), mode="bilinear", align_corners=False)
    return up.reshape(*lead, H, W)


def make_case(V, H, W, n, seed, coarse=1, behind=True):
    """(points [n,3], img_ref, renderings, w2c, ixt): points in a cube larger than the object, so that some fall partly
    or wholly outside a view, plus (behind=True) points behind each camera."""
    g = torch.Generator().manual_seed(seed)
    cams, w2c, ixt = lara_cameras(V, H, W, seed)
    img_ref = _field(g, (V, 3, H, W), H, W, coarse)
    image = _field(g, (V, 3, H, W), H, W, coarse).permute(0, 2, 3, 1).contiguous()
    acc = _field(g, (V, H, W), H, W, coarse)
    depth = (1.905 + (_field(g, (V, H, W), H, W, coarse) - 0.5)).unsqueeze(-1)
    points = (torch.rand((n, 3), generator=g) - 0.5) * 2.0
    if behind:
        k = min(n, 4 * V)          # points behind camera v: beyond its centre, seen from the origin
        for j in range(k):
            c = cams[j % V].c2w[:3, 3]
            points[(j * 7919) % n] = c * (1.2 + 0.1 * (j // V)) + 0.05 * torch.randn(3, generator=g)
    return points, img_ref, {"image": image, "acc_map": acc, "depth": depth}, w2c, ixt


# ---- CPU: restatement vs LaRa's own code ----------------------------------------------------------------------
V_CPU, H_CPU, W_CPU, N_CPU = 3, 48, 64, 2600


def _cpu_case():
    points, img_ref, rend, w2c, ixt = make_case(V_CPU, H_CPU, W_CPU, N_CPU, 11)
    g = torch.Generator().manual_seed(12)
    mask = torch.rand(N_CPU, generator=g) < 0.77
    up = torch.randn((V_CPU, 8, int(mask.sum())), generator=g)
    return points, mask, img_ref, rend, w2c, ixt, up


def _grads_record(feats, pts, r):
    return {"feats": fingerprint(feats.detach().numpy()), "g_points": fingerprint(pts.grad.numpy()),
            **{"g_" + k: fingerprint(v.grad.numpy()) for k, v in r.items()}}


def record_reference(lara, dev):
    """LaRa's own get_point_feats on the CPU (run this file as a script to write the record)."""
    net = _import_reference_network(lara)
    points, mask, img_ref, rend, w2c, ixt, up = _cpu_case()
    pts = points.clone().requires_grad_(True)
    r = {k: v.clone().requires_grad_(True) for k, v in rend.items()}
    fake_self = types.SimpleNamespace(device=torch.device(dev))
    batch = {"tar_w2c": w2c[None], "tar_ixt": ixt[None]}
    feats, _ = net.Network.get_point_feats(fake_self, 0, img_ref, r, V_CPU, batch, pts, mask)
    feats.backward(up)
    return {"point_feats": _grads_record(feats, pts, r)}


def test_point_feats_restatement_matches_reference_on_cpu():
    points, mask, img_ref, rend, w2c, ixt, up = _cpu_case()
    pts = points.clone().requires_grad_(True)
    r = {k: v.clone().requires_grad_(True) for k, v in rend.items()}
    feats = point_feats_torch(pts[mask], img_ref, r, w2c, ixt)
    feats.backward(up)
    assert _grads_record(feats, pts, r) == reference_record("test_point_feats", "point_feats")


# ---- CPU: argument checks ----------------------------------------------------------------------------------------
def _small(dtype=torch.float32):
    points, img_ref, rend, w2c, ixt = make_case(2, 8, 10, 5, 3, behind=False)
    return (points.to(dtype), img_ref.to(dtype), {k: v.to(dtype) for k, v in rend.items()}, w2c.to(dtype), ixt.to(dtype))


@pytest.mark.parametrize("what", ["points", "img_ref", "image", "acc_map", "depth", "w2c", "ixt"])
def test_sample_point_feats_rejects_bad_shapes(what):
    from lara_b200.point_feats import sample_point_feats
    points, img_ref, rend, w2c, ixt = _small()
    bad = {"points": lambda: (points[:, :2], img_ref, rend, w2c, ixt),
           "img_ref": lambda: (points, img_ref[:, :2], rend, w2c, ixt),
           "image": lambda: (points, img_ref, {**rend, "image": rend["image"].permute(0, 3, 1, 2)}, w2c, ixt),
           "acc_map": lambda: (points, img_ref, {**rend, "acc_map": rend["acc_map"][:, :-1]}, w2c, ixt),
           "depth": lambda: (points, img_ref, {**rend, "depth": rend["depth"][..., 0]}, w2c, ixt),
           "w2c": lambda: (points, img_ref, rend, w2c[:1], ixt),
           "ixt": lambda: (points, img_ref, rend, w2c, ixt[:, :2])}[what]()
    with pytest.raises(RuntimeError, match="sample_point_feats"):
        sample_point_feats(*bad)


def test_sample_point_feats_rejects_dtype_device_and_constants_requiring_grad():
    from lara_b200.point_feats import sample_point_feats
    with pytest.raises(RuntimeError, match="Float"):
        sample_point_feats(*_small(torch.float64))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        sample_point_feats(*_small())
    with pytest.raises(KeyError):
        points, img_ref, rend, w2c, ixt = _small()
        sample_point_feats(points, img_ref, {"image": rend["image"], "depth": rend["depth"]}, w2c, ixt)
    for k in range(3):
        points, img_ref, rend, w2c, ixt = _small()
        consts = [img_ref, w2c, ixt]
        consts[k] = consts[k].clone().requires_grad_(True)
        with pytest.raises(RuntimeError, match="requires grad"):
            sample_point_feats(points, consts[0], rend, consts[1], consts[2])


def test_point_feats_c_entries_reject_bad_arguments(lib):
    P = ctypes.c_void_p(256)           # never dereferenced: the checks come before any CUDA call
    ins = [P] * 7
    for V, n, H, W in ((0, 4, 8, 8), (1, -1, 8, 8), (1, 4, 0, 8), (1, 4, 8, 0)):
        assert lib.srf_point_feats_forward(None, V, n, H, W, *ins, P) != 0
        assert b"srf_point_feats_forward: bad sizes" in lib.srf_last_error()
        assert lib.srf_point_feats_backward(None, V, n, H, W, *ins, P, P, P, P, P) != 0
        assert b"srf_point_feats_backward: bad sizes" in lib.srf_last_error()
    for k in range(7):
        nulled = list(ins)
        nulled[k] = None
        assert lib.srf_point_feats_forward(None, 1, 4, 8, 8, *nulled, P) != 0
        assert b"null input pointer" in lib.srf_last_error()
        assert lib.srf_point_feats_backward(None, 1, 4, 8, 8, *nulled, P, None, None, None, None) != 0
        assert b"null input pointer" in lib.srf_last_error()
    assert lib.srf_point_feats_forward(None, 1, 4, 8, 8, *ins, None) != 0
    assert b"null output pointer" in lib.srf_last_error()
    assert lib.srf_point_feats_backward(None, 1, 4, 8, 8, *ins, None, P, P, P, P) != 0
    assert b"null upstream gradient" in lib.srf_last_error()
    # n == 0: nothing to read or write, so the empty point set's pointers may be NULL
    assert lib.srf_point_feats_forward(None, 1, 0, 8, 8, None, *ins[1:], None) == 0
    assert lib.srf_point_feats_backward(None, 1, 0, 8, 8, None, *ins[1:], None, None, None, None, None) == 0


# ---- GPU: kernel vs restatement ----------------------------------------------------------------------------------
def restated_coords(points, w2c, ixt, H, W):
    """[V,n,2] grid_sample source coordinates (ix, iy) along the restatement's own chain of fp32 operations."""
    cam = points.reshape(1, -1, 3) @ w2c[:, :3, :3].permute(0, 2, 1) + w2c[:, :3, 3][:, None]
    cam = cam @ ixt.permute(0, 2, 1)
    wh = torch.tensor([W, H], device=points.device)
    g = (cam[..., :2] / cam[..., -1:] + 0.5) / wh * 2 - 1.0
    return ((g + 1) * wh - 1) / 2


def near_jump(coords, H, W, eps=1e-3):
    """[V,n] bool: in that view a coordinate of the point that reaches the image lies within eps px of a pixel-centre
    line, where the point gradient jumps.  Pixel centres sit at integer source coordinates; the lines -1 and size,
    where the outermost taps enter or leave the image border, are integers too."""
    size = torch.tensor([W, H], dtype=coords.dtype, device=coords.device)
    c = coords.double()
    reaches = torch.isfinite(c) & (c > -1 - eps) & (c < size + eps)
    return (reaches & ((c - c.round()).abs() <= eps)).any(-1)


def _run(fn, points, img_ref, rend, w2c, ixt, up):
    pts = points.clone().requires_grad_(True)
    r = {k: v.clone().requires_grad_(True) for k, v in rend.items()}
    out = fn(pts, img_ref, r, w2c, ixt)
    out.backward(up)
    return out.detach(), pts.grad, {k: v.grad for k, v in r.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("V,n,H,W", [(4, 262144, 512, 512), (2, 1000, 80, 96), (1, 1, 32, 32)])
def test_point_feats_kernel_matches_restatement(cuda_device, V, n, H, W):
    from lara_b200.point_feats import sample_point_feats
    dev = cuda_device
    points, img_ref, rend, w2c, ixt = make_case(V, H, W, n, n, coarse=8)
    points, img_ref, w2c, ixt = points.to(dev), img_ref.to(dev), w2c.to(dev), ixt.to(dev)
    rend = {k: v.to(dev) for k, v in rend.items()}
    up = torch.randn((V, 8, n), generator=torch.Generator().manual_seed(n + 1)).to(dev)
    f1, gp1, gr1 = _run(sample_point_feats, points, img_ref, rend, w2c, ixt, up)
    f2, gp2, gr2 = _run(point_feats_torch, points, img_ref, rend, w2c, ixt, up)
    assert f1.shape == f2.shape == (V, 8, n) and gp1.shape == (n, 3)
    for c in range(8):
        assert rel_err(f1[:, c].cpu().numpy(), f2[:, c].cpu().numpy()) < 1e-5, c
    for k in gr1:
        assert gr1[k].shape == gr2[k].shape, k
        assert rel_err(gr1[k].cpu().numpy(), gr2[k].cpu().numpy()) < 1e-5, k
    if n > 1:      # at least one view each: outside, partly outside, behind a camera
        ix = restated_coords(points, w2c, ixt, H, W)
        z = (points @ w2c[:, 2, :3].T + w2c[:, 2, 3]).T
        assert bool((z < 0).any()), "no point behind a camera"
        inside = ((ix > 0) & (ix < torch.tensor([W - 1, H - 1], device=dev))).all(-1)
        assert bool((~inside).any()) and bool(inside.any())
    # A point's gradient sums its views, so a point is left out if it is near a line in any view.  Each of the 2V
    # coordinates of a point that reaches every view is within 1e-3 px of a line with probability 2e-3, so at V = 4
    # about 1.6 % of such points go; the bound is on the (point, view) pairs left out.
    near = near_jump(restated_coords(points, w2c, ixt, H, W), H, W)
    keep = ~near.any(0)
    assert float(near.float().mean()) < 0.01
    assert rel_err(gp1[keep].cpu().numpy(), gp2[keep].cpu().numpy()) < 1e-4


@pytest.mark.gpu
def test_point_feats_empty_point_set(cuda_device):
    from lara_b200.point_feats import sample_point_feats
    dev = cuda_device
    points, img_ref, rend, w2c, ixt = make_case(2, 16, 24, 1, 4, behind=False)
    rend = {k: v.to(dev) for k, v in rend.items()}
    out, gp, gr = _run(sample_point_feats, points[:0].to(dev), img_ref.to(dev), rend, w2c.to(dev), ixt.to(dev),
                       torch.zeros((2, 8, 0), device=dev))
    assert out.shape == (2, 8, 0) and gp.shape == (0, 3)
    for k, v in gr.items():
        assert v.shape == rend[k].shape and not bool(v.any()), k


@pytest.mark.gpu
def test_point_in_camera_plane_samples_zero(cuda_device):
    """A point with z = 0 in a source view samples 0 and gets no gradient; the other points are unaffected."""
    from lara_b200.point_feats import sample_point_feats
    dev = cuda_device
    H, W, n = 40, 56, 300
    points, img_ref, rend, _, ixt = make_case(1, H, W, n, 9, behind=False)
    w2c = torch.eye(4)[None].clone()
    w2c[0, 2, 3] = 2.0                 # camera at z = -2 looking down +z: z_cam = z + 2 exactly
    z0 = 150
    points[z0] = torch.tensor([0.3, -0.2, -2.0])
    up = torch.randn((1, 8, n), generator=torch.Generator().manual_seed(3))
    rend = {k: v.to(dev) for k, v in rend.items()}
    args = (img_ref.to(dev), rend, w2c.to(dev), ixt[:1].to(dev))
    f, gp, gr = _run(sample_point_feats, points.to(dev), *args, up.to(dev))
    assert not bool(f[:, :, z0].any()) and not bool(gp[z0].any())
    others = torch.arange(n) != z0
    f_o, gp_o, gr_o = _run(sample_point_feats, points[others].to(dev), *args, up[:, :, others].to(dev))
    assert torch.equal(f[:, :, others.to(dev)], f_o) and torch.equal(gp[others.to(dev)], gp_o)
    for k in gr:
        assert rel_err(gr[k].cpu().numpy(), gr_o[k].cpu().numpy()) < 1e-6, k


@pytest.mark.gpu
def test_point_feats_gradient_reaches_the_rasterizer(cuda_device):
    """render_scene_views -> sample_point_feats on the first views -> scalar of features and coarse outputs ->
    backward: the Gaussian-parameter gradients match those through the restatement."""
    from lara_b200 import rasterizer as R
    from lara_b200 import scene as S
    from lara_b200.multiview import render_scene_views
    from lara_b200.point_feats import sample_point_feats
    dev = cuda_device
    P, H, W, V, n_sel = 20000, 128, 128, 6, 4
    sc = S.scene(P, 3)
    cams, w2c, ixt = lara_cameras(V, H, W, 3)
    settings = [S.settings_for(c, torch.ones(3), sc["sh_degree"], dev, R.GaussianRasterizationSettings) for c in cams]
    g = torch.Generator().manual_seed(6)
    rays = torch.cat([torch.zeros(V, H, W, 3), torch.nn.functional.normalize(torch.randn((V, H, W, 3), generator=g), dim=-1)], -1).to(dev)
    img_ref = torch.rand((n_sel, 3, H, W), generator=g).to(dev)
    mask = (torch.rand(P, generator=g) < 0.5).to(dev)
    w_feat = torch.randn((n_sel, 8, int(mask.sum())), generator=g).to(dev)
    w_out = {k: torch.randn(s, generator=g).to(dev) for k, s in (("image", (V, H, W, 3)), ("depth", (V, H, W, 1)),
                                                                  ("acc_map", (V, H, W)))}
    grads = []
    for fn in (sample_point_feats, point_feats_torch):
        leaves = {k: sc[k].to(dev).clone().requires_grad_(True) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
        out = render_scene_views(leaves["means3D"], leaves["shs"], leaves["opacities"], leaves["scales"],
                                 leaves["rotations"], settings, rays=rays)
        rend = {k: out[k][:n_sel] for k in ("image", "acc_map", "depth")}
        feats = fn(leaves["means3D"][mask], img_ref, rend, w2c[:n_sel].to(dev), ixt[:n_sel].to(dev))
        loss = (feats * w_feat).sum() + sum((out[k] * w).sum() for k, w in w_out.items())
        loss.backward()
        grads.append({k: leaves[k].grad.detach().cpu().numpy() for k in ("shs", "opacities", "scales", "rotations")})
    for k in grads[0]:
        assert rel_err(grads[0][k], grads[1][k]) < 1e-4, k


if __name__ == "__main__":
    # python tests/test_point_feats.py OUT_DIR LARA_CHECKOUT: record LaRa's outputs, as tests/golden/make_reference_records.py
    # does for the other modules
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_reference_records import save
    out_dir, lara = sys.argv[1:3]
    os.makedirs(out_dir, exist_ok=True)
    save(out_dir, "test_point_feats", record_reference(lara, "cpu"))
