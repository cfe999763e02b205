"""LaRa's ``Network`` on the fused path (DESIGN §3.28) on an H100, at LaRa's size: B = 3 scenes of V = 8 target views
of 512^2, n_views_sel = 4, P = 524288 Gaussians per scene (LaRa's base config), seeded weights.  The masks the fine
pass checks are LaRa's opacity cut in scene 0, forced empty in scene 1 (``_check_mask``'s sparse branch) and full in
scene 2 (its dense branch, in training mode).

* cameras: ``batch_cameras``' view matrix equals the float64 inverse rounded to fp32 or lies one ulp from it, for
  rigid and for scaled, sheared poses; campos, bg and the padding are bit for bit; a singular and a NaN pose render
  their background only; the distance from LaRa's ``MiniCam`` (``torch.inverse`` on the device) is reported and bounded;
* no arithmetic added: ``Network.forward(with_fine=True)`` equals, bit for bit, the stage calls composed by hand on the
  same records (outputs and ``render_pkg``) and LaRa's per-scene loop through ``render_scene_views`` /
  ``render_subset_views``;
* the step ``Losses()(batch, net(batch, with_fine=True), 5000)`` and its backward under
  ``torch.use_deterministic_algorithms(True)``: every parameter gradient equals the composed stages' bit for bit, and
  two runs give the same bits; without the fine pass the fine head gets no gradient and every other parameter does;
* bf16 autocast (fp32 outputs, equal to the composed stages under autocast) and ``no_grad`` (the same bits, no node);
* torch-visible synchronising calls of the forward: the top read plus ``FineSubset``'s reads, pinned.
"""
import gc
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

pytestmark = pytest.mark.gpu

B, V, H, W, NVS = 3, 8, 512, 512, 4
KEYS = ("image", "depth", "acc_map", "rend_normal", "depth_normal", "rend_dist")
# |record - MiniCam| per view-matrix element, relative to the matrix's largest entry: torch's fp32 inverse is within a
# few ulps of the correctly rounded one
MINICAM_BOUND = 2.0 ** -20


def _forced(sig):
    """LaRa's opacity cut in scene 0; scene 1 all below it (sparse branch), scene 2 all above (dense branch)."""
    out = sig.clone()
    out[1] = 0.0
    out[2] = 1.0
    return out


@pytest.fixture(scope="module")
def setup():
    from bench_network import base_cfg, lara_batch
    from lara_b200.network import Network
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    net = Network(base_cfg(NVS)).to(dev).train()
    net.gs_render.opacity_activation = lambda o: _forced(torch.sigmoid(o))
    with torch.no_grad():        # splats near LaRa's initial voxel-sized scale, not the seeded head's wide spread
        net.decoder.mlp_coarse[4].weight.mul_(0.1)
    gc.collect()
    torch.cuda.empty_cache()
    yield net, lara_batch(dev), dev
    del net
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(autouse=True)
def _release():
    """Each case starts from the memory the module holds: graphs of earlier cases that cycles keep alive are freed."""
    gc.collect()
    torch.cuda.empty_cache()
    yield


def _run(net, batch, with_fine=True, return_buffer=False, seed=7):
    torch.manual_seed(seed)
    return net(batch, with_fine=with_fine, return_buffer=return_buffer)


def composed(net, batch, with_fine=True, seed=7):
    """Network.forward's stage calls written out by hand on the same records."""
    from lara_b200.batch import batch_cameras
    from lara_b200.multiview import BatchCameras, FineSubset, render_batch_subset_views, render_batch_views
    from lara_b200.point_feats import sample_batch_point_feats
    torch.manual_seed(seed)
    tar = batch["tar_rgb"]
    inps = tar[:, :NVS].reshape(B * NVS, H, W, 3).permute(0, 3, 1, 2)
    feats = net.img_encoder.forward_maps(inps)
    fv, coarse, fine = net._feat_volume(), net._stages["coarse"], net._stages["fine"]
    rays, w2cs, ixts = (batch[k][:, :NVS] for k in ("tar_rays_down", "tar_w2c", "tar_ixt"))
    vol = net.vol_decoder([fv.cond_tokens(feats, rays, w2cs, ixts, (H, W), g) for g in net.n_groups])
    g = coarse.gaussians(vol, net.group_centers, net.opacity_shift, net.scaling_shift, 0.5 * 0.5 / 32)
    centers, shs, scaling, rotation, opacity = g
    masks = _forced(torch.sigmoid(opacity).squeeze(-1)) > 0.005
    fov = batch["fovx"].tolist()
    cams = BatchCameras(batch_cameras(batch["tar_c2w"], batch["bg_color"]), H, W,
                        [(math.tan(f * 0.5),) * 2 for f in fov], 1)
    out = render_batch_views(centers, shs, opacity, scaling, rotation, rays=batch["tar_rays"], raw_activations=True,
                             keep_binning=True, cameras=cams)
    res = {k: out[k] for k in KEYS}
    extra = {"gaussians": g, "cams": cams, "out": out}
    if with_fine:
        sub = FineSubset(masks, check=True, training=net.training)
        pf = sample_batch_point_feats(sub, centers, tar[:, :NVS].permute(0, 1, 4, 2, 3), out, w2cs, ixts)
        shs_fine = fine.fine_shs(vol.view(B, -1, 80), 2, sub, pf, shs)
        of = render_batch_subset_views(out["binning"], sub, shs_fine)
        res.update({k + "_fine": of[k + "_fine"] for k in KEYS})
        extra.update(sub=sub, shs_fine=shs_fine, vol=vol)
    return res, extra


def _same(a, b, what):
    assert a.dtype == b.dtype and a.shape == b.shape, (what, a.dtype, b.dtype, a.shape, b.shape)
    assert torch.equal(a, b), (what, float((a.double() - b.double()).abs().max()))


# ---- cameras ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rigid", [True, False])
def test_camera_records(rigid):
    from test_network import camera_record64, exact_view_f32, poses
    from lara_b200.batch import batch_cameras
    from bench_network import MiniCam
    dev = torch.device("cuda:0")
    c2w = poses(B * V * 8, 11 if rigid else 12, rigid)
    bg = np.random.default_rng(2).choice([0.0, 0.5, 1.0], (len(c2w), 3)).astype(np.float32)
    got = batch_cameras(torch.from_numpy(c2w).to(dev).view(-1, V, 4, 4), torch.from_numpy(bg).to(dev).view(-1, V, 3))
    got = got.cpu().numpy()
    want = camera_record64(c2w, bg)
    assert np.array_equal(got[:, 16:], want[:, 16:])
    want[:, :16] = exact_view_f32(c2w)
    ulps = np.abs(got[:, :16].view(np.int32).astype(np.int64) - want[:, :16].view(np.int32).astype(np.int64))
    same_sign = np.sign(got[:, :16]) == np.sign(want[:, :16])
    # one ulp, or, for an entry that fp64 cancellation leaves far below the matrix's scale, within fp64 rounding of it
    near_zero = np.abs(got[:, :16].astype(np.float64) - want[:, :16]) <= 2.0 ** -46 * np.abs(want[:, :16]).max(1, keepdims=True)
    one_ulp = ((ulps <= 1) & same_sign) | (got[:, :16] == want[:, :16])
    assert (one_ulp | near_zero).all(), int(ulps.max())
    print(f"[cameras] entries beyond one ulp (all within fp64 rounding of the scale): {int((~one_ulp).sum())} of "
          f"{one_ulp.size}")
    lara = []
    for c, b in zip(torch.from_numpy(c2w).to(dev), torch.from_numpy(bg).to(dev)):
        cam = MiniCam(c, W, H, torch.tensor(0.6, device=dev), torch.tensor(0.6, device=dev), 1.2, 2.8, dev)
        lara.append(torch.cat([cam.world_view_transform.reshape(16), cam.camera_center, b, torch.zeros(2, device=dev)]))
    lara = torch.stack(lara).cpu().numpy()
    assert np.array_equal(got[:, 16:], lara[:, 16:])
    scale = np.abs(got[:, :16]).max(axis=1, keepdims=True)
    dist = float((np.abs(got[:, :16].astype(np.float64) - lara[:, :16]) / scale).max())
    print(f"[cameras] rigid={rigid}: max |record - MiniCam| / max|viewmatrix| = {dist:.3e} (bound {MINICAM_BOUND:.1e})")
    assert dist <= MINICAM_BOUND


def test_bad_poses_render_background_only():
    from bench_network import lara_batch
    from lara_b200.batch import batch_cameras
    from lara_b200.multiview import BatchCameras, render_batch_views
    dev = torch.device("cuda:0")
    d = lara_batch(dev, B=1, V=4, H=64, W=64, seed=3)
    c2w = d["tar_c2w"].clone()
    c2w[0, 1, :3, :3] = 0.0                       # singular
    c2w[0, 2, 1, 2] = float("nan")                # NaN
    d["bg_color"][0, 1] = torch.tensor([0.25, 0.5, 1.0], device=dev)
    d["bg_color"][0, 2] = torch.tensor([1.0, 0.0, 0.5], device=dev)
    cams = batch_cameras(c2w, d["bg_color"])
    assert torch.isfinite(cams).all()
    g = torch.Generator(device=dev).manual_seed(0)
    P = 4096
    centers = (torch.rand(1, P, 3, generator=g, device=dev) - 0.5) * 0.6
    shs = torch.rand(1, P, 4, 3, generator=g, device=dev)
    opacity = torch.full((1, P, 1), 2.0, device=dev)
    scales, rot = torch.full((1, P, 2), -3.0, device=dev), torch.rand(1, P, 4, generator=g, device=dev)
    out = render_batch_views(centers, shs, opacity, scales, rot, rays=d["tar_rays"], raw_activations=True,
                             cameras=BatchCameras(cams, 64, 64, [(math.tan(0.3),) * 2], 1))
    for v in (1, 2):
        assert torch.equal(out["image"][0, v], d["bg_color"][0, v].expand(64, 64, 3)), v
        assert float(out["acc_map"][0, v].abs().max()) == 0.0
        assert bool((out["radii"][0, v] == 0).all())
    for v in (0, 3):          # the good views see the Gaussians
        assert float(out["acc_map"][0, v].max()) > 0.5


# ---- the forward -----------------------------------------------------------------------------------------------------
def test_forward_equals_composed_stages_and_lara_loop(setup):
    from lara_b200.multiview import render_scene_views, render_subset_views
    from lara_b200.point_feats import sample_point_feats
    from lara_b200.rasterizer import GaussianRasterizationSettings
    net, batch, dev = setup
    with torch.no_grad():
        out = _run(net, batch, return_buffer=True)
        ref, ex = composed(net, batch)
    assert set(out) == set(ref) | {"render_pkg"}
    for k in ref:
        _same(out[k], ref[k], k)
        assert out[k].shape[:2] == (B, V)
    sub = ex["sub"]
    assert sub.counts[1] > 0 and sub.counts[2] < sub.P, sub.counts      # both _check_mask branches fired
    pkg = out["render_pkg"]
    assert len(pkg) == 2 * B
    centers, shs, scaling, rotation, opacity = ex["gaussians"]
    for b in range(B):
        for got, want in zip(pkg[2 * b], (centers[b], shs[b], opacity[b], scaling[b], rotation[b])):
            _same(got, want, f"coarse pkg {b}")
        mask = sub.masks[b]
        lo, hi = sub.offsets[b], sub.offsets[b + 1]
        fine = (centers[b][mask], ex["shs_fine"][lo:hi], opacity[b], scaling[b], rotation[b], mask)
        for got, want in zip(pkg[2 * b + 1], fine):
            _same(got, want, f"fine pkg {b}")
    # LaRa's per-scene loop on the same records: one scene at a time, its views' settings carrying the records
    cams = ex["cams"].cams
    tanf = math.tan(float(batch["fovx"][0]) * 0.5)
    for b in range(B):
        sets = [GaussianRasterizationSettings(
            image_height=H, image_width=W, tanfovx=tanf, tanfovy=tanf, bg=cams[b * V + j, 19:22], scale_modifier=1.0,
            viewmatrix=cams[b * V + j, :16].view(4, 4), projmatrix=torch.eye(4, device=dev), sh_degree=1,
            campos=cams[b * V + j, 16:19], prefiltered=False, debug=False) for j in range(V)]
        with torch.no_grad():
            o = render_scene_views(centers[b], shs[b], opacity[b], scaling[b], rotation[b], sets,
                                   rays=batch["tar_rays"][b], raw_activations=True, keep_binning=True)
            mask = sub.masks[b]
            src = {k: o[k][:NVS] for k in ("image", "acc_map", "depth")}          # rendering_coarse: the source views
            pf = sample_point_feats(centers[b][mask], batch["tar_rgb"][b, :NVS].permute(0, 3, 1, 2), src,
                                    batch["tar_w2c"][b, :NVS], batch["tar_ixt"][b, :NVS])
            sf = net._stages["fine"].fine_shs(ex["vol"].view(B, -1, 80)[b], 2, mask, pf, shs[b])
            of = render_subset_views(o["binning"], mask, sf)
        for k in KEYS:
            _same(out[k][b], o[k], f"loop {k} {b}")
            _same(out[k + "_fine"][b], of[k + "_fine"], f"loop {k}_fine {b}")


def _grads(net):
    return {n: (None if p.grad is None else p.grad.clone()) for n, p in net.named_parameters()}


def test_step_gradients_are_the_composed_stages_and_deterministic(setup):
    from lara_b200.loss import Losses
    net, batch, _ = setup
    torch.use_deterministic_algorithms(True)
    try:
        runs = []
        for _ in range(2):
            net.zero_grad(set_to_none=True)
            Losses()(batch, _run(net, batch), 5000)[0].backward()
            runs.append(_grads(net))
        net.zero_grad(set_to_none=True)
        Losses()(batch, composed(net, batch)[0], 5000)[0].backward()
        ref = _grads(net)
    finally:
        torch.use_deterministic_algorithms(False)
    for n, g in ref.items():
        assert g is not None, n
        _same(runs[0][n], g, n)
        _same(runs[1][n], g, n)


def test_without_fine_pass_the_fine_head_gets_no_gradient(setup):
    from lara_b200.loss import Losses
    net, batch, _ = setup
    net.zero_grad(set_to_none=True)
    out = _run(net, batch, with_fine=False)
    assert not any(k.endswith("_fine") for k in out)
    Losses()(batch, out, 5000)[0].backward()
    for n, p in net.named_parameters():
        fine = n.startswith(("decoder.norm.", "decoder.cross_att.", "decoder.mlp_fine."))
        assert (p.grad is None) == fine, n
    net.zero_grad(set_to_none=True)


def test_bf16_autocast(setup):
    from lara_b200.loss import Losses
    net, batch, _ = setup
    net.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = _run(net, batch)
        loss = Losses()(batch, out, 5000)[0]
        with torch.no_grad():
            ref = composed(net, batch)[0]
    loss.backward()
    assert all(p.grad is not None for p in net.parameters())
    for k in ref:
        assert out[k].dtype == torch.float32, k
        _same(out[k].detach(), ref[k], k)
    net.zero_grad(set_to_none=True)


def test_no_grad_same_bits_no_node(setup):
    net, batch, _ = setup
    with_grad = _run(net, batch)
    assert all(v.grad_fn is not None for v in with_grad.values())
    with_grad = {k: v.detach() for k, v in with_grad.items()}
    gc.collect()
    with torch.no_grad():
        without = _run(net, batch)
    for k in with_grad:
        assert without[k].grad_fn is None and not without[k].requires_grad, k
        _same(without[k], with_grad[k], k)


def test_host_syncs(setup):
    from test_gpu_fine_pass_batch import _count_syncs
    net, batch, _ = setup
    torch.cuda.synchronize()
    with torch.no_grad():
        n_fine, where = _count_syncs(lambda: _run(net, batch))
        torch.cuda.synchronize()
        n_coarse, where_c = _count_syncs(lambda: _run(net, batch, with_fine=False))
    torch.cuda.synchronize()
    # the top read of the per-scene field of view and size; FineSubset's count read, and its second one because a
    # _check_mask branch fired
    assert n_coarse == 1, where_c
    assert n_fine == 3, where
