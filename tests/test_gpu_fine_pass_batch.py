"""LaRa's fine pass over all B scenes of a batch in three calls (DESIGN §3.26) against the per-scene loop it replaces.

At LaRa's size (B = 3, 8 target views of 512^2, the first Vs = 4 the source views, P = 524288 = 64^3 voxels x K = 2,
SH degree 1, D = 80) with LaRa's opacity cut in scene 0, an empty scene 1 and a full scene 2:

* forward: ``sample_batch_point_feats``, the batch form of ``FineHead.fine_shs`` and ``render_batch_subset_views``
  with a ``FineSubset`` equal the per-scene ``sample_point_feats`` / ``fine_shs`` calls and the mask-tensor render
  bit for bit; ``img_ref`` read in place from a channel-last ``tar_rgb`` view gives the bits of a planar copy;
* backward under ``torch.use_deterministic_algorithms(True)``: the gradients of the centers, the coarse renderings,
  ``volume_feat_up`` and ``shs_coarse`` equal the loop's bit for bit; the fine head's parameter gradients are within
  1e-5 of each tensor's maximum, and two batched runs give identical bits;
* default mode: each scene's rendering and point gradients lie within ``oracle/point_feats64.py``'s per-element bound;
* at most one torch-visible synchronising op for the batched fine pass when no ``_check_mask`` branch fires, two when
  one does; S = 1 of the scene entries is the one-scene entry; an all-empty batch and B = 1 work.
"""
import os
import warnings

import pytest
import torch

from lara_b200.fine_head import FineHead
from lara_b200.multiview import FineSubset, render_batch_subset_views, render_batch_views
from lara_b200.point_feats import sample_batch_point_feats, sample_point_feats
from test_gpu_batch_views import _batch
from test_point_feats import make_case
from test_point_feats_per_element import _planar, _upstream, check_all, statement

pytestmark = pytest.mark.gpu

B, V, VS, H, W = 3, 8, 4, 512, 512
N, K, D, SH_DIM = 64 ** 3, 2, 80, 12
P = N * K
FINE_KEYS = tuple(k + "_fine" for k in ("image", "depth", "acc_map", "rend_normal", "depth_normal", "rend_dist"))


def _cameras(settings, dev):
    """w2c [B,Vs,4,4] and pinhole ixt [B,Vs,3,3] of the first Vs views of each scene (focal from the field of view,
    principal point at the centre, as LaRa's loader builds them)."""
    w2c = torch.stack([torch.stack([s.viewmatrix.T for s in sc[:VS]]) for sc in settings]).contiguous()
    ixt = torch.zeros(B, VS, 3, 3)
    for b, sc in enumerate(settings):
        fx, fy = W / (2 * float(sc[0].tanfovx)), H / (2 * float(sc[0].tanfovy))
        ixt[b, :, 0, 0], ixt[b, :, 1, 1], ixt[b, :, 0, 2], ixt[b, :, 1, 2], ixt[b, :, 2, 2] = fx, fy, W / 2, H / 2, 1
    return w2c.to(dev), ixt.to(dev)


@pytest.fixture(scope="module")
def lara_batch(cuda_device):
    dev = cuda_device
    params, settings, rays, _ = _batch(B, V, P, 41, dev)
    g = torch.Generator(device="cuda").manual_seed(5)
    tar_rgb = torch.rand(B, V, H, W, 3, generator=g, device=dev)
    vf = torch.randn(B, N, D, generator=g, device=dev)
    masks = (torch.sigmoid(params[2]) > 0.005).view(B, P)     # LaRa's opacity cut
    masks[1] = False
    masks[2] = True
    head = FineHead(D, SH_DIM).to(dev)
    torch.manual_seed(0)
    for p in head.parameters():
        p.data.add_(torch.randn(p.shape, device=dev) * 0.05)
    w2c, ixt = _cameras(settings, dev)
    return dict(params=params, settings=settings, rays=rays, tar_rgb=tar_rgb, vf=vf, masks=masks, head=head, w2c=w2c,
                ixt=ixt)


def _fine_pass(d, batched, det, seed=3):
    """One coarse render, then the fine pass (batched or LaRa's per-scene loop) and the backward of a seeded weighted
    sum of the fine outputs to the leaves.  Returns the outputs, the gradients and the intermediate results."""
    dev = d["vf"].device
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        leaves = [p.detach().clone().requires_grad_(True) for p in d["params"]]
        vf = d["vf"].detach().clone().requires_grad_(True)
        head = d["head"]
        head.zero_grad(set_to_none=True)
        out = render_batch_views(*leaves, d["settings"], rays=d["rays"], raw_activations=True, keep_binning=True)
        for k in ("image", "acc_map", "depth"):
            out[k].retain_grad()
        img_ref = d["tar_rgb"][:, :VS].permute(0, 1, 4, 2, 3)        # LaRa's _inps, channel-last, read in place
        centers, shs_coarse = leaves[0], leaves[1]
        if batched:
            sub = FineSubset(d["masks"])
            pf = sample_batch_point_feats(sub, centers, img_ref, out, d["w2c"], d["ixt"])
            shs = head.fine_shs(vf, K, sub, pf, shs_coarse)
            fine = render_batch_subset_views(out["binning"], sub, shs)
        else:
            pfs, shs_l = [], []
            for b in range(B):
                m = d["masks"][b]
                rend = {k: out[k][b][:VS] for k in ("image", "acc_map", "depth")}
                pf = sample_point_feats(centers[b][m], img_ref[b], rend, d["w2c"][b], d["ixt"][b])
                # the one-scene head takes no empty mask (LaRa's _check_mask never leaves one): nothing to compute
                shs_l.append(head.fine_shs(vf[b], K, m, pf, shs_coarse[b]) if m.any() else shs_coarse[b][:0])
                pfs.append(pf)
            pf, shs = torch.cat(pfs, 2), torch.cat(shs_l)
            fine = render_batch_subset_views(out["binning"], d["masks"], shs)
        g = torch.Generator(device="cuda").manual_seed(seed)
        loss = sum((fine[k] * torch.randn(fine[k].shape, generator=g, device=dev)).sum() for k in FINE_KEYS)
        loss.backward()
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev)
    grads = {"centers": leaves[0].grad, "shs_coarse": leaves[1].grad, "opacity": leaves[2].grad,
             "scales": leaves[3].grad, "rotations": leaves[4].grad, "volume_feat_up": vf.grad}
    grads.update({"coarse_" + k: out[k].grad for k in ("image", "acc_map", "depth")})
    params = {n: p.grad.clone() for n, p in head.named_parameters()}
    return dict(pf=pf.detach(), shs=shs.detach(), fine={k: fine[k].detach() for k in FINE_KEYS}, grads=grads,
                params=params)


@pytest.fixture(scope="module")
def det_runs(lara_batch):
    return {"loop": _fine_pass(lara_batch, False, True), "batch": _fine_pass(lara_batch, True, True),
            "batch2": _fine_pass(lara_batch, True, True)}


def test_masks_cover_the_cases(lara_batch):
    c = lara_batch["masks"].sum(1).tolist()
    assert 0 < c[0] < P and c[1] == 0 and c[2] == P


def test_forward_bit_for_bit(det_runs):
    a, b = det_runs["loop"], det_runs["batch"]
    assert torch.equal(a["pf"], b["pf"])
    assert torch.equal(a["shs"], b["shs"])
    for k in FINE_KEYS:
        assert torch.equal(a["fine"][k], b["fine"][k]), k


def test_backward_deterministic_bit_for_bit(det_runs):
    a, b, b2 = det_runs["loop"], det_runs["batch"], det_runs["batch2"]
    for k in a["grads"]:
        assert torch.equal(a["grads"][k], b["grads"][k]), k
        assert torch.equal(b["grads"][k], b2["grads"][k]), k
    for k, ref in a["params"].items():
        scale = float(ref.double().abs().max())
        err = float((b["params"][k].double() - ref.double()).abs().max())
        assert err <= 1e-5 * scale, (k, err, scale)
        assert torch.equal(b["params"][k], b2["params"][k]), k


def test_img_ref_in_place_equals_planar_copy(lara_batch):
    d = lara_batch
    sub = FineSubset(d["masks"])
    with torch.no_grad():
        out = render_batch_views(*d["params"], d["settings"], rays=d["rays"], raw_activations=True)
        strided = d["tar_rgb"][:, :VS].permute(0, 1, 4, 2, 3)
        assert not strided.is_contiguous()
        a = sample_batch_point_feats(sub, d["params"][0], strided, out, d["w2c"], d["ixt"])
        b = sample_batch_point_feats(sub, d["params"][0], strided.contiguous(), out, d["w2c"], d["ixt"])
    assert torch.equal(a, b)


def test_one_scene_entry_is_s1_of_the_scene_entry(cuda_device):
    pts, img_ref, rend, w2c, ixt = make_case(3, 64, 80, 2000, 4, coarse=4)
    dev = cuda_device
    up = _upstream(3, 2000, 9).to(dev)
    for det in (False, True):
        prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(det)
        try:
            p1 = pts.to(dev).requires_grad_(True)
            r1 = {k: v.to(dev).requires_grad_(True) for k, v in rend.items()}
            f1 = sample_point_feats(p1, img_ref.to(dev), r1, w2c.to(dev), ixt.to(dev))
            f1.backward(up)
            p2 = pts.to(dev)[None].clone().requires_grad_(True)
            r2 = {k: v.to(dev)[None].clone().requires_grad_(True) for k, v in rend.items()}
            sub = FineSubset(torch.ones(1, 2000, dtype=torch.bool, device=dev))
            f2 = sample_batch_point_feats(sub, p2, img_ref.to(dev)[None], r2, w2c.to(dev)[None], ixt.to(dev)[None])
            f2.backward(up)
        finally:
            torch.use_deterministic_algorithms(prev)
        assert torch.equal(f1, f2)
        assert torch.equal(p1.grad, p2.grad[0])
        if det:
            for k in r1:
                assert torch.equal(r1[k].grad, r2[k].grad[0]), k


def test_default_mode_within_float64_bound(cuda_device):
    """Three scenes of the per-element cases at sizes the float64 statement handles, one of them empty, each scene's
    columns and gradient rows against its own statement."""
    dev = cuda_device
    Vs, Hs, Ws, Pp = 2, 80, 96, 1200
    counts = (1000, 0, 700)
    cases = [make_case(Vs, Hs, Ws, max(c, 1), 20 + b, coarse=8) for b, c in enumerate(counts)]
    centers = torch.zeros(3, Pp, 3)
    masks = torch.zeros(3, Pp, dtype=torch.bool)
    for b, c in enumerate(counts):
        rows = torch.arange(c) * (Pp // max(c, 1))
        centers[b, rows] = cases[b][0][:c]
        masks[b, rows] = True
    img_ref = torch.stack([c[1] for c in cases]).to(dev)
    rend = {k: torch.stack([c[2][k] for c in cases]).to(dev).requires_grad_(True) for k in ("image", "acc_map", "depth")}
    w2c, ixt = torch.stack([c[3] for c in cases]).to(dev), torch.stack([c[4] for c in cases]).to(dev)
    sub = FineSubset(masks.to(dev))
    cen = centers.to(dev).requires_grad_(True)
    ups = [_upstream(Vs, c, 30 + b) for b, c in enumerate(counts)]
    up = torch.cat(ups, 2).to(dev)
    feats = sample_batch_point_feats(sub, cen, img_ref, rend, w2c, ixt)
    feats.backward(up)
    torch.cuda.synchronize()
    for b, c in enumerate(counts):
        o0, o1 = sub.offsets[b], sub.offsets[b + 1]
        gi, ga, gd = _planar({"image": rend["image"].grad[b], "acc_map": rend["acc_map"].grad[b],
                              "depth": rend["depth"].grad[b]})
        rows = masks[b].nonzero()[:, 0]
        assert float(cen.grad[b][~masks[b]].abs().max()) == 0.0
        if c == 0:
            assert not gi.any() and not ga.any() and not gd.any()
            continue
        case = (cases[b][0][:c],) + tuple(cases[b][1:])
        st = statement(case, ups[b])
        res = {"feats": feats[:, :, o0:o1].detach().cpu().numpy(), "g_points": cen.grad[b][rows].cpu().numpy(),
               "g_image": gi, "g_acc": ga, "g_depth": gd}
        check_all(res, st, False, f"scene {b}")


def _count_syncs(fn):
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    hits = [x for x in w if "called a synchronizing cuda operation" in str(x.message).lower()]
    return len(hits), [f"{os.path.basename(x.filename)}:{x.lineno}" for x in hits]


@pytest.mark.parametrize("branch", [False, True])
def test_host_syncs(lara_batch, branch):
    d = lara_batch
    masks = d["masks"].clone()
    if not branch:
        masks[1, :100000] = True              # no empty scene: without training, no branch fires
    with torch.no_grad():
        out = render_batch_views(*d["params"], d["settings"], rays=d["rays"], raw_activations=True, keep_binning=True)
        img_ref = d["tar_rgb"][:, :VS].permute(0, 1, 4, 2, 3)
        out["binning"].state.resolve()
        torch.cuda.synchronize()

        def fine():
            sub = FineSubset(masks, check=True, training=False)
            pf = sample_batch_point_feats(sub, d["params"][0], img_ref, out, d["w2c"], d["ixt"])
            shs = d["head"].fine_shs(d["vf"], K, sub, pf, d["params"][1])
            render_batch_subset_views(out["binning"], sub, shs)
        fine()                                    # first-call set-up is not part of the steady state
        torch.cuda.synchronize()
        n, where = _count_syncs(fine)
    print(f"\n  torch-visible synchronising ops, branch={branch}: {n} at {where}")
    assert n <= (2 if branch else 1)


def test_all_empty_batch_and_one_scene(lara_batch):
    d = lara_batch
    dev = d["vf"].device
    img_ref = d["tar_rgb"][:, :VS].permute(0, 1, 4, 2, 3)
    out = render_batch_views(*[p.detach() for p in d["params"]], d["settings"], rays=d["rays"], raw_activations=True)
    out = {k: out[k] for k in ("image", "acc_map", "depth")}
    centers = d["params"][0].detach().clone().requires_grad_(True)
    sub = FineSubset(torch.zeros(B, P, dtype=torch.bool, device=dev))
    pf = sample_batch_point_feats(sub, centers, img_ref, out, d["w2c"], d["ixt"])
    assert pf.shape == (VS, 8, 0)
    shs = d["head"].fine_shs(d["vf"], K, sub, pf, d["params"][1])
    assert shs.shape == (0, SH_DIM // 3, 3)
    pf.sum().backward()
    assert not centers.grad.any()
    # B = 1: scene 0 alone against the one-scene calls
    m = d["masks"][:1]
    sub1 = FineSubset(m)
    one = {k: out[k][:1] for k in out}
    pf1 = sample_batch_point_feats(sub1, d["params"][0][:1], img_ref[:1], one, d["w2c"][:1], d["ixt"][:1])
    ref = sample_point_feats(d["params"][0][0][m[0]], img_ref[0], {k: out[k][0][:VS] for k in out}, d["w2c"][0],
                             d["ixt"][0])
    assert torch.equal(pf1, ref)
    s1 = d["head"].fine_shs(d["vf"][:1], K, sub1, pf1, d["params"][1][:1])
    assert torch.equal(s1, d["head"].fine_shs(d["vf"][0], K, m[0], ref, d["params"][1][0]))
