"""LaRa's fine pass rendered from the coarse pass's binning (``render_subset_views``, DESIGN §3.18) against the gathered
render it replaces (``render_scene_views(c[mask], shs_fine, o[mask], s[mask], r[mask], ...)``): outputs, tile lists and
records bit for bit, gradients bit for bit in deterministic mode, and LaRa's fine chain end to end."""
import warnings

import pytest
import torch

from lara_b200 import rasterizer as R
from lara_b200 import scene as S
from lara_b200.debug import unpack_state
from lara_b200.multiview import OUT_KEYS, _subset_forward, render_scene_views, render_subset_views
from test_chain_per_element import N_SEL, _pinhole, lara_rays

KEYS = OUT_KEYS + ("radii",)


def _case(P, V, H, W, deg, raw, seed, dev, far=0, big=False):
    """A LaRa-like scene (raw network outputs when `raw`), V cameras with LaRa's rays, and new SH coefficients for every
    Gaussian.  `far` Gaussians are moved out of every view (culled); `big` makes every splat large (instances overflow
    the first capacity guess)."""
    sc = S.scene(P, seed, deg)
    c, shs, o, s, r = sc["means3D"], sc["shs"], sc["opacities"], sc["scales"], sc["rotations"]
    if far:
        c[:far] = torch.tensor([40.0, -35.0, 50.0])
    if big:
        s = s * 12.0
    if raw:
        o, s, r = torch.logit(o), torch.log(s), r * 1.7
    cams = S.cameras(V, H, W, seed)
    bg = torch.tensor([0.25, 0.5, 1.0])
    settings = [S.settings_for(cm, bg, deg, dev, R.GaussianRasterizationSettings) for cm in cams]
    rays = torch.stack([lara_rays(cm) for cm in cams]).to(dev)
    g = torch.Generator().manual_seed(seed + 5)
    shs_new = torch.randn(shs.shape, generator=g) * 0.6
    return [t.to(dev).contiguous() for t in (c, shs, o, s, r)], settings, rays, shs_new.to(dev)


def _mask(kind, params, raw, seed):
    c, _, o, _, _ = params
    P = c.shape[0]
    opac = torch.sigmoid(o) if raw else o
    lara = opac.view(-1) > 0.005
    g = torch.Generator(device=c.device).manual_seed(seed)
    if kind == "lara":
        return lara
    if kind == "half":          # the training half-drop of LaRa's _check_mask on top of the opacity cut
        return lara & (torch.rand((P,), generator=g, device=c.device) < 0.5)
    if kind == "all":
        return torch.ones(P, dtype=torch.bool, device=c.device)
    if kind == "none":
        return torch.zeros(P, dtype=torch.bool, device=c.device)
    if kind == "single":
        m = torch.zeros(P, dtype=torch.bool, device=c.device)
        m[P // 3] = True
        return m
    if kind == "culled":        # every culled (far) Gaussian and a random third of the rest
        m = torch.rand((P,), generator=g, device=c.device) < 0.33
        m[:64] = True
        return m
    raise ValueError(kind)


def _both(params, settings, rays, raw, mask, shs_new, grad):
    c, shs, o, s, r = [t.detach().requires_grad_(grad) for t in params]
    out = render_scene_views(c, shs, o, s, r, settings, rays=rays, raw_activations=raw, keep_binning=True)
    shs_fine = shs_new[mask].contiguous()
    sub = render_subset_views(out["binning"], mask, shs_fine)
    ref = render_scene_views(c[mask], shs_fine, o[mask], s[mask], r[mask], settings, rays=rays, raw_activations=raw,
                             prex="_fine")
    return out, sub, ref


def _assert_equal(sub, ref, ctx):
    assert set(sub) == set(ref), ctx
    for k in KEYS:
        a, b = sub[k + "_fine"], ref[k + "_fine"]
        assert a.shape == b.shape and torch.equal(a, b), f"{ctx} {k}"


@pytest.mark.gpu
@pytest.mark.parametrize("P,V,H,W,deg,raw,masks", [
    (524288, 8, 512, 512, 1, True, ("lara", "half", "all")),
    (524288, 8, 512, 512, 3, False, ("half",)),
    (40000, 3, 203, 317, 0, True, ("lara", "half", "all", "none", "single", "culled")),
    (40000, 3, 203, 317, 2, False, ("half", "single", "culled")),
    (40000, 2, 203, 317, 3, True, ("half", "none")),
    (40000, 2, 64, 48, 1, False, ("lara", "all", "none", "culled")),
])
def test_forward_bit_identity(cuda_device, P, V, H, W, deg, raw, masks):
    params, settings, rays, shs_new = _case(P, V, H, W, deg, raw, P + H + deg, cuda_device, far=64)
    for kind in masks:
        mask = _mask(kind, params, raw, deg + 3)
        _, sub, ref = _both(params, settings, rays, raw, mask, shs_new, grad=True)
        _assert_equal(sub, ref, f"{kind} P={P} {H}x{W} deg={deg} raw={raw}")
        assert sub["image_fine"].grad_fn is not None


@pytest.mark.gpu
@pytest.mark.parametrize("raw,coarse_grad", [(True, True), (False, False)])
def test_lists_and_records(cuda_device, raw, coarse_grad):
    P, V, H, W, deg = 60000, 3, 203, 317, 2
    params, settings, rays, shs_new = _case(P, V, H, W, deg, raw, 11, cuda_device, far=64)
    c, shs, o, s, r = [t.detach().requires_grad_(coarse_grad) for t in params]
    mask = _mask("half", params, raw, 4)
    idx = mask.nonzero().view(-1)
    n = idx.numel()
    out = render_scene_views(c, shs, o, s, r, settings, rays=rays, raw_activations=raw, keep_binning=True)
    b = out["binning"]
    shs_fine = shs_new[idx].contiguous()
    _, (_, _, st) = _subset_forward(b, idx, shs_fine, True)
    cams = R.pack_cameras(settings, cuda_device)
    _, _, radii, fresh = R.forward_views_raw(c[idx].detach(), shs_fine, None, o[idx].detach(), s[idx].detach(),
                                             r[idx].detach(), None, cams, settings[0].tanfovx, settings[0].tanfovy, H, W,
                                             deg, raw_activations=raw)
    torch.cuda.synchronize()
    for v in range(V):
        us, uf = unpack_state(st, n, H, W, view=v), unpack_state(fresh, n, H, W, view=v)
        vis = radii[v] > 0
        assert int(vis.sum()) < n
        assert torch.equal(us["rect"], uf["rect"])
        assert torch.equal(us["rec"][vis].view(torch.int32), uf["rec"][vis].view(torch.int32)), v
        assert torch.equal(us["depths"][vis].view(torch.int32), uf["depths"][vis].view(torch.int32)), v
        rs, rf = us["ranges"].cpu(), uf["ranges"].cpu()
        ps, pf = us["point_list"].cpu(), uf["point_list"].cpu()
        assert torch.equal(rs[:, 1] - rs[:, 0], rf[:, 1] - rf[:, 0]), v
        for t in torch.nonzero(rf[:, 1] > rf[:, 0]).view(-1).tolist():
            assert torch.equal(ps[rs[t, 0]:rs[t, 1]], pf[rf[t, 0]:rf[t, 1]]), (v, t)


def _grads(params, settings, rays, raw, mask, shs_new, subset, seed):
    c, shs, o, s, r = [t.detach().requires_grad_(True) for t in params]
    shs_fine = shs_new[mask].contiguous().requires_grad_(True)
    if subset:
        out = render_scene_views(c, shs, o, s, r, settings, rays=rays, raw_activations=raw, keep_binning=True)
        fine = render_subset_views(out["binning"], mask, shs_fine)
    else:
        fine = render_scene_views(c[mask], shs_fine, o[mask], s[mask], r[mask], settings, rays=rays,
                                  raw_activations=raw, prex="_fine")
    g = torch.Generator(device=c.device).manual_seed(seed)
    loss = sum((fine[k + "_fine"] * torch.randn(fine[k + "_fine"].shape, generator=g, device=c.device)).sum()
               for k in OUT_KEYS)
    loss.backward()
    torch.cuda.synchronize()
    return [c.grad, o.grad, s.grad, r.grad, shs_fine.grad]


@pytest.mark.gpu
@pytest.mark.parametrize("P,V,H,W,deg,raw,kind", [
    (524288, 8, 512, 512, 1, True, "half"), (40000, 3, 203, 317, 3, False, "culled"),
    (40000, 3, 203, 317, 0, True, "none"), (40000, 3, 203, 317, 2, True, "single")])
def test_gradients(cuda_device, P, V, H, W, deg, raw, kind):
    params, settings, rays, shs_new = _case(P, V, H, W, deg, raw, P + deg, cuda_device, far=64)
    mask = _mask(kind, params, raw, 9)
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        a = _grads(params, settings, rays, raw, mask, shs_new, True, 1)
        b = _grads(params, settings, rays, raw, mask, shs_new, False, 1)
        for i, (x, y) in enumerate(zip(a, b)):
            if y is None:       # n = 0: the gathered render treats the empty SH tensor as absent and gives it no grad
                assert kind == "none" and i == 4 and x.numel() == 0
                continue
            assert x.shape == y.shape and torch.equal(x, y), i
        torch.use_deterministic_algorithms(False)
        a = _grads(params, settings, rays, raw, mask, shs_new, True, 1)
    finally:
        torch.use_deterministic_algorithms(prev)
    for i, (x, y) in enumerate(zip(a, b)):      # default mode: the bound tests/test_deterministic.py uses
        if y is None:
            continue
        assert x.shape == y.shape, i
        if y.numel():
            assert float((x - y).abs().max()) <= 1e-5 * float(y.abs().max()), i
    if kind == "none":
        assert all(float(x.abs().max()) == 0.0 for x in a[:4])
    else:
        assert float(a[0][~mask].abs().max()) == 0.0 and float(a[0][mask].abs().max()) > 0.0


def _fine_chain(dev, subset):
    """coarse render (raw activations, LaRa rays) -> sample_point_feats on the first N_SEL views -> FineHead.fine_shs
    -> fine render -> scene_loss(prex="_fine") added to the coarse loss, one backward in deterministic mode."""
    from lara_b200.loss import scene_loss
    from lara_b200.point_feats import sample_point_feats
    from test_fine_head import _head
    N, K_, sh_dim, V, H, W = 9000, 2, 12, 3, 168, 144
    params, settings, rays, _ = _case(N * K_, V, H, W, 1, True, 77, dev)
    cams = S.cameras(V, H, W, 77)
    g = torch.Generator().manual_seed(79)
    tar = torch.rand((V, H, W, 3), generator=g).to(dev)
    mask = (torch.rand((N * K_,), generator=g) < 0.5).to(dev)
    img_ref = torch.rand((N_SEL, 3, H, W), generator=g).to(dev)
    vf = (torch.randn((N, 80), generator=g) * 0.5 + 0.3).to(dev).requires_grad_(True)
    head = _head(80, sh_dim, 13, dev)
    w2c, ixt = (t.to(dev) for t in _pinhole(cams))
    c, shs, o, s, r = [t.detach().requires_grad_(True) for t in params]
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        out = render_scene_views(c, shs, o, s, r, settings, rays=rays, raw_activations=True, keep_binning=subset)
        loss, _ = scene_loss(out, tar, 5000)
        pf = sample_point_feats(c[mask], img_ref, {k: out[k][:N_SEL] for k in ("image", "acc_map", "depth")},
                                w2c[:N_SEL], ixt[:N_SEL])
        shs_fine = head.fine_shs(vf, K_, mask, pf, shs)
        if subset:
            fine = render_subset_views(out["binning"], mask, shs_fine)
        else:
            fine = render_scene_views(c[mask], shs_fine, o[mask], s[mask], r[mask], settings, rays=rays,
                                      raw_activations=True, prex="_fine")
        loss_fine, _ = scene_loss(fine, tar, 5000, prex="_fine")
        (loss + loss_fine).backward()
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev)
    return [float(loss_fine)] + [t.grad for t in (c, shs, o, s, r, vf)] + [p.grad for p in head.parameters()]


@pytest.mark.gpu
def test_lara_fine_chain(cuda_device):
    a, b = _fine_chain(cuda_device, True), _fine_chain(cuda_device, False)
    assert a[0] == b[0]
    for i, (x, y) in enumerate(zip(a[1:], b[1:])):
        assert (x is None) == (y is None), i
        assert x is None or torch.equal(x, y), i


@pytest.mark.gpu
@pytest.mark.parametrize("ctx", ["no_grad", "inference_mode", "plain"])
def test_forward_only(cuda_device, ctx):
    """Forward-only subset renders, on a coarse state of the autograd path and on a forward-only coarse state, are
    bit-identical to the gathered render and create no autograd node."""
    params, settings, rays, shs_new = _case(40000, 3, 203, 317, 1, True, 5, cuda_device, far=64)
    mask = _mask("half", params, True, 2)
    out_g, _, ref = _both(params, settings, rays, True, mask, shs_new, grad=True)
    subs = []
    if ctx == "plain":         # nothing requires grad
        subs.append(_both(params, settings, rays, True, mask, shs_new, grad=False)[1])
    else:
        with (torch.no_grad if ctx == "no_grad" else torch.inference_mode)():
            subs.append(render_subset_views(out_g["binning"], mask, shs_new[mask]))
            out_f = render_scene_views(*params, settings, rays=rays, raw_activations=True, keep_binning=True)
            assert not out_f["binning"].state.for_backward
            subs.append(render_subset_views(out_f["binning"], mask, shs_new[mask]))
    for sub in subs:
        _assert_equal(sub, ref, ctx)
        assert sub["image_fine"].grad_fn is None


@pytest.mark.gpu
def test_coarse_overflow(cuda_device):
    """A scene of large splats overflows the first capacity guess: the coarse stage 2 is re-run before the lists are
    filtered, and the subset render still equals the gathered one."""
    R._capacity_hwm.clear()
    params, settings, rays, shs_new = _case(20000, 2, 256, 256, 1, True, 21, cuda_device, big=True)
    mask = _mask("half", params, True, 3)
    c, shs, o, s, r = [t.detach().requires_grad_(True) for t in params]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        out = render_scene_views(c, shs, o, s, r, settings, rays=rays, raw_activations=True, keep_binning=True)
        st = out["binning"].state
        cap0 = st.capacity
        shs_fine = shs_new[mask].contiguous()
        sub = render_subset_views(out["binning"], mask, shs_fine)
    assert st.capacity > cap0, "the case must overflow the first capacity"
    ref = render_scene_views(c[mask], shs_fine, o[mask], s[mask], r[mask], settings, rays=rays, raw_activations=True,
                             prex="_fine")
    _assert_equal(sub, ref, "overflow")


@pytest.mark.gpu
def test_bad_inputs_raise(cuda_device):
    params, settings, rays, shs_new = _case(5000, 2, 64, 64, 1, True, 3, cuda_device)
    c, shs, o, s, r = [t.detach().requires_grad_(True) for t in params]
    mask = _mask("half", params, True, 1)
    n = int(mask.sum())
    out = render_scene_views(c, shs, o, s, r, settings, rays=rays, raw_activations=True, keep_binning=True)
    b = out["binning"]
    with pytest.raises(RuntimeError, match="mask"):
        render_subset_views(b, mask.int(), shs_new[mask])
    with pytest.raises(RuntimeError, match="mask"):
        render_subset_views(b, mask[:-1], shs_new[mask])
    with pytest.raises(RuntimeError, match="mask"):
        render_subset_views(b, mask.cpu(), shs_new[mask])
    with pytest.raises(RuntimeError, match="shs_fine"):
        render_subset_views(b, mask, shs_new[mask][:, :3])
    with pytest.raises(RuntimeError, match="shs_fine"):
        render_subset_views(b, mask, shs_new[mask][: n - 1])
    with pytest.raises(RuntimeError, match="shs_fine"):
        render_subset_views(b, mask, shs_new[mask].double())
    with pytest.raises(TypeError):
        render_subset_views(out, mask, shs_new[mask])
    with torch.no_grad():
        o.add_(0.0)
    with pytest.raises(RuntimeError, match="modified in place"):
        render_subset_views(b, mask, shs_new[mask])
