"""The kernels around the rasterizer in LaRa's training step, element by element, against float64 with a bound per element.

The fused ``render_img`` epilogue (csrc/epilogue.cu), the loss producer (csrc/loss.cu) and the decoder layout
(csrc/decoder.cu) are restated in float64 by ``oracle.chain64``, each value carrying a bound on what an fp32 evaluation of
the same formula may differ by (the blend replay's per-operation rules, ``oracle.oracle.EB``).  So a gradient is
checked on its own scale: ``dL/dD = g / alpha`` where alpha is small, the four-neighbour sum that carries the
pseudo-normal gradient into the depth, and a small offset gradient are each held to their own bound, not to a fraction
of the tensor's largest element.

CPU part: the float64 statements equal the plain-torch restatements (pinned to LaRa's own code) run in float64, and the
fp32 restatements lie within the bound.  GPU part: the kernels against the statements, on renderings with LaRa's rays
(every ray starts at the camera centre, so empty pixels back-project to one point), on synthetic maps for the edges,
and along the whole chain decoder -> renderer -> loss -> backward, link by link.
"""
import numpy as np
import pytest
import torch

from oracle import chain64 as C
from oracle.oracle import EB, K

f64 = np.float64
OUT_KEYS = ("image", "depth", "acc_map", "rend_normal", "depth_normal", "rend_dist")
FLOOR64 = 2.0 ** -29          # the bound with double's 2^-52 per operation in place of fp32's 2^-23


def _planar(t):
    t = t.detach().cpu() if hasattr(t, "detach") else torch.as_tensor(t)
    return (t.permute(2, 0, 1) if t.ndim == 3 else t).numpy()


def _compare(got, ref: EB, excl=None, ctx=""):
    """|got - ref| <= bound at every element outside `excl` (a mask over the trailing [H,W], or of ref's shape).
    Returns the worst err/bound."""
    a = np.asarray(got, f64).reshape(ref.v.shape)
    err = np.abs(a - ref.v)
    keep = np.ones(ref.v.shape, bool) if excl is None else ~np.broadcast_to(np.asarray(excl, bool), ref.v.shape)
    with np.errstate(invalid="ignore"):
        bad = ~(err <= ref.e) & keep & np.isfinite(ref.e)          # an infinite bound: checked for properties
        ratio = np.where(keep & (err > 0), err / np.where(ref.e > 0, ref.e, np.inf), 0.0)
    ratio = np.where(np.isfinite(ref.e), ratio, 0.0)
    where = None
    if bad.any():
        idx = tuple(int(i) for i in np.argwhere(bad)[0])
        where = (idx, float(a[idx]), float(ref.v[idx]), float(ref.e[idx]))
    assert not bad.any(), f"{ctx}: {int(bad.sum())} of {bad.size} elements outside their bound, first at {where}"
    return float(ratio.max()) if ratio.size else 0.0


def _pin64(got, ref: EB, ctx=""):
    """A float64 evaluation of the same formula: within 1e-12 relative plus the double-rounding floor of the bound."""
    a = np.asarray(got, f64).reshape(ref.v.shape)
    fin = np.isfinite(ref.e)
    err = np.abs(a - ref.v)
    ok = err <= 1e-12 * np.abs(ref.v) + FLOOR64 * ref.e
    assert (ok | ~fin).all(), f"{ctx}: {int((~ok & fin).sum())} elements differ, worst {float(err[fin].max()):.3g}"


def _tightness(name, ref: EB):
    """Median and 90th percentile of bound / |value| over the non-zero finite elements: a vacuous bound shows."""
    m = (np.abs(ref.v) > 0) & np.isfinite(ref.e)
    r = ref.e[m] / np.abs(ref.v[m])
    if r.size:
        print(f"  {name}: bound/|value| median {np.median(r):.3g}, p90 {np.percentile(r, 90):.3g}")
        return float(np.median(r))
    return 0.0


# ---------------------------------------------------------------------------------------------------------- inputs

def lara_rays(cam):
    """LaRa's build_rays (dataLoader/utils.py): the camera centre as the origin of every pixel's ray, the direction
    K^-1 (u + 0.5, v + 0.5, 1) rotated into the world (not normalised)."""
    H, W = cam.image_height, cam.image_width
    fx, fy = W / (2 * cam.tanfovx), H / (2 * cam.tanfovy)
    c2w = cam.c2w.double()
    X, Y = torch.meshgrid(torch.arange(W, dtype=torch.float64), torch.arange(H, dtype=torch.float64), indexing="xy")
    d = torch.stack([(X + 0.5 - W / 2) / fx, (Y + 0.5 - H / 2) / fy, torch.ones_like(X)], -1) @ c2w[:3, :3].T
    return torch.cat([c2w[:3, 3].expand(H, W, 3), d], -1).float().contiguous()


def synthetic(H, W, seed, overflow=False, bad_median=False):
    """An epilogue input with the edges LaRa's renderings have: background (alpha == 0), a silhouette, one-pixel-wide
    rows and columns of coverage, isolated covered pixels, colour exactly 0 and 1 and beyond both; optionally alpha
    so small that D / alpha overflows fp32 (not float64), alpha and D so small that alpha * alpha underflows while D / alpha
    is an ordinary depth, and NaN / +-inf median depths.  LaRa's rays."""
    from lara_b200 import scene as S
    rng = np.random.default_rng(seed)
    cam = S.cameras(1, H, W, seed)[0]
    yy, xx = np.mgrid[0:H, 0:W]
    alpha = np.zeros((H, W), np.float32)
    disc = (yy - 0.45 * H) ** 2 + (xx - 0.55 * W) ** 2 < (0.3 * min(H, W)) ** 2
    alpha[disc] = rng.uniform(0.3, 1.0, int(disc.sum()))
    alpha[H // 5, :] = rng.uniform(0.2, 1.0, W)                   # a one-pixel-wide row
    alpha[:, W // 6] = rng.uniform(0.2, 1.0, H)                   # ... and column
    iso = rng.integers(0, H * W, max(1, H * W // 40))             # isolated covered pixels
    alpha.reshape(-1)[iso] = rng.uniform(0.05, 1.0, iso.size)
    depth = (1.9 + 0.2 * np.sin(yy / 5.0) * np.cos(xx / 7.0) + 0.01 * rng.standard_normal((H, W))).astype(np.float32)
    allmap = np.zeros((8, H, W), np.float32)
    allmap[0] = depth * alpha
    allmap[1] = alpha
    n = rng.standard_normal((3, H, W)).astype(np.float32)
    allmap[2:5] = n / np.linalg.norm(n, axis=0) * alpha
    allmap[5] = np.where(alpha > 0, depth + 0.02 * rng.standard_normal((H, W)), 0).astype(np.float32)
    allmap[6] = (1e-3 * rng.random((H, W)) * alpha).astype(np.float32)
    allmap[7] = rng.random((H, W)).astype(np.float32)
    if overflow:
        k = rng.choice(np.flatnonzero(alpha.reshape(-1) > 0), max(1, H * W // 50))
        allmap[1].reshape(-1)[k] = np.float32(1e-39)              # subnormal: fp32(D) / alpha overflows
        allmap[0].reshape(-1)[k] = np.float32(2.0)
        k = rng.choice(np.flatnonzero(alpha.reshape(-1) > 0), max(1, H * W // 50))
        allmap[1].reshape(-1)[k] = np.float32(1e-25)              # D / alpha finite, alpha * alpha underflows
        allmap[0].reshape(-1)[k] = (np.float32(1e-25) * depth.reshape(-1)[k]).astype(np.float32)
    if bad_median:
        k = rng.integers(0, H * W, max(3, H * W // 30))
        allmap[5].reshape(-1)[k] = np.array([np.nan, np.inf, -np.inf], np.float32)[np.arange(k.size) % 3]
    color = (rng.random((3, H, W)) * 1.4 - 0.2).astype(np.float32)
    color.reshape(-1)[rng.integers(0, 3 * H * W, max(2, H * W // 10))] = 0.0
    color.reshape(-1)[rng.integers(0, 3 * H * W, max(2, H * W // 10))] = 1.0
    vm = cam.viewmatrix.numpy().reshape(16)
    return color, allmap, lara_rays(cam).numpy(), vm


def upstreams(H, W, seed, only=None):
    """Planar upstream gradients of the six outputs, magnitude ~1; `only` keeps one."""
    rng = np.random.default_rng(seed)
    shapes = {"image": (3, H, W), "depth": (H, W), "acc_map": (H, W), "rend_normal": (3, H, W),
              "depth_normal": (3, H, W), "rend_dist": (H, W)}
    return {k: (rng.standard_normal(s).astype(np.float32) if only in (None, k) else None) for k, s in shapes.items()}


def _vjp(st, ups):
    return C.epilogue_vjp64(None, None, None, None, None, ups["image"], ups["depth"], ups["acc_map"],
                            ups["rend_normal"], ups["depth_normal"], ups["rend_dist"], state=st)


# ------------------------------------------------------------------------------------------------------ CPU: the pins

def _torch_epilogue(color, allmap, rays, vm, depth_ratio, ups, dtype):
    from oracle.torch_restatements import render_img_epilogue_torch
    c = torch.from_numpy(color).to(dtype).requires_grad_(True)
    a = torch.from_numpy(allmap).to(dtype).requires_grad_(True)
    out = render_img_epilogue_torch(c, a, torch.from_numpy(rays).to(dtype), torch.from_numpy(vm).reshape(4, 4).to(dtype),
                                    depth_ratio)
    loss = (c * 0).sum() + (a * 0).sum()
    for k, v in out.items():
        if ups[k] is not None:
            g = torch.from_numpy(ups[k]).to(dtype)
            loss = loss + ((v.permute(2, 0, 1) if v.ndim == 3 else v) * g).sum()
    loss.backward()
    return {k: _planar(v) for k, v in out.items()}, c.grad.numpy(), a.grad.numpy()


@pytest.mark.parametrize("depth_ratio", [0.0, 0.5, 1.0])
@pytest.mark.parametrize("edges", [False, True])
def test_epilogue64_pins(depth_ratio, edges):
    """epilogue64 / epilogue_vjp64 == render_img_epilogue_torch in float64 (the D / alpha gradients where D / alpha is
    finite: torch's is NaN at alpha == 0; every other channel is compared there too), and the fp32 restatement lies within the
    bound.  `edges`: overflowing D / alpha, alpha and D so small that alpha * alpha underflows, and non-finite medians,
    where only the fp32 restatement takes the kernel's decisions."""
    color, allmap, rays, vm = synthetic(29, 38, 3, overflow=edges, bad_median=edges)
    ups = upstreams(29, 38, 4)
    st = C.EpilogueState(color, allmap, rays, vm, depth_ratio)
    out, band, inf = C.epilogue64(None, None, None, None, None, state=st)
    dc, da, excl = _vjp(st, ups)
    assert band.sum() == 0
    # torch's D / alpha gradient (channels 0, 1) is NaN wherever fp32 D / alpha is not finite (0 * inf in autograd):
    # at alpha == 0, and where it overflows; its median gradient (channel 5) is NaN at a non-finite median whose
    # surface-depth gradient is NaN (0 * NaN).  The kernel writes 0 at both, by the same decisions.
    nan_ok = np.zeros(allmap.shape, bool)
    nan_ok[:2] = ~st.q_ok
    nan_ok[5] = ~st.m_ok
    print(f"\nepilogue pins depth_ratio={depth_ratio} edges={edges}: infinite-bound pixels {int(inf.sum())}")
    if not edges:
        o64, gc64, ga64 = _torch_epilogue(color, allmap, rays, vm, depth_ratio, ups, torch.float64)
        for k in OUT_KEYS:
            _pin64(o64[k], out[k], k)
        _pin64(gc64, dc, "d_color")
        _pin64(np.where(nan_ok, 0.0, ga64), EB(np.where(nan_ok, 0.0, da.v), da.e), "d_allmap")
        assert np.isnan(ga64[:2][nan_ok[:2]]).all()            # the difference the kernel documents
    o32, gc32, ga32 = _torch_epilogue(color, allmap, rays, vm, depth_ratio, ups, torch.float32)
    worst = 0.0
    for k in OUT_KEYS:
        worst = max(worst, _compare(o32[k], out[k], ctx=k))
        _tightness(k, out[k])
    worst = max(worst, _compare(gc32, dc, ctx="d_color"))
    worst = max(worst, _compare(ga32, da, np.broadcast_to(excl, nan_ok.shape) | nan_ok, "d_allmap"))
    _tightness("d_allmap", da)
    print(f"  fp32 restatement: worst err/bound {worst:.3g}")


def _loss_case(V, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(s, generator=g)                    # noqa: E731
    n = lambda *s: torch.nn.functional.normalize(r(*s) - 0.5, dim=1)     # noqa: E731
    return {"image": r(V, 3, H, W), "rend_normal": n(V, 3, H, W), "depth_normal": n(V, 3, H, W),
            "acc_map": r(V, H, W), "rend_dist": r(V, H, W) * 0.01}, r(V, H, W, 3)


@pytest.mark.parametrize("it", [1000, 1001])
def test_loss64_pins(it):
    """loss64 == lara_loss_torch in float64 over a batch of B = 2 scenes (values and gradients for an upstream of 3);
    the fp32 restatement's gradient maps and stats lie within the bound.  The sums' bound follows loss_sums_kernel's
    reduction tree, not torch's: that the fp32 restatement's means lie within it says nothing about the tree; that the
    kernel's sums do is checked on the GPU (test_loss_per_element)."""
    from lara_b200.multiview import concat_views
    from oracle.torch_restatements import lara_loss_torch
    B, V, H, W, up = 2, 3, 16, 24, 3.0
    scenes = [_loss_case(V, H, W, 10 + b) for b in range(B)]
    with_reg = it > 1000
    res = {}
    for dtype in (torch.float64, torch.float32):
        leaves = [{k: v.to(dtype).requires_grad_(True) for k, v in pl.items()} for pl, _ in scenes]
        cl = lambda d: {k: (v.permute(0, 2, 3, 1) if v.ndim == 4 else v) for k, v in d.items()}     # noqa: E731
        outs = [concat_views(cl(d)) for d in leaves]
        batch = {k: torch.stack([o[k] for o in outs]) for k in outs[0]}
        tar = torch.stack([t for _, t in scenes]).to(dtype)
        loss, stats = lara_loss_torch(batch, tar, it)
        (loss * up).backward()
        res[dtype] = (float(loss.detach()), {k: float(v) for k, v in stats.items()}, leaves)
    tot = 0.0
    stat = {k: (0.0, 0.0) for k in (("mse", "distortion", "normal") if with_reg else ("mse",))}
    for b, (pl, tar) in enumerate(scenes):
        vals, grads = C.loss64(pl["image"], tar, pl["rend_normal"], pl["depth_normal"], pl["acc_map"], pl["rend_dist"],
                               with_reg, B, up, blocks=1)
        tot += vals["loss"][0]
        for k, g in grads.items():
            g64, g32 = res[torch.float64][2][b][k].grad, res[torch.float32][2][b][k].grad
            if g is None:
                assert g64 is None or float(g64.abs().max()) == 0.0, k
                continue
            _pin64(g64.numpy(), g, k)
            print(f"  {k}: fp32 restatement worst err/bound {_compare(g32.numpy(), g, ctx=k):.3g}")
            _tightness(k, g)
        for k in stat:
            stat[k] = (stat[k][0] + vals[k][0], stat[k][1] + vals[k][1])
    assert abs(res[torch.float64][0] - tot) <= 1e-12 * abs(tot)
    for k, (v, e) in stat.items():      # the scenes' shares; the fp32 restatement's mean rounds once more
        assert abs(res[torch.float32][1][k] - v) <= e + 0.5 * K * abs(v), k
        assert abs(res[torch.float64][1][k] - v) <= 1e-12 * abs(v), k


def _decoder_case(B, N, K_, sh_dim, seed):
    g = torch.Generator().manual_seed(seed)
    C_ = 10 + sh_dim
    feats = torch.randn((B, N, K_ * C_), generator=g) * 3
    grid = torch.rand((N, 3), generator=g) - 0.5
    return feats, grid


def test_decoder64_pins():
    from oracle.torch_restatements import decoder_layout_torch
    feats, grid = _decoder_case(2, 300, 2, 12, 0)
    g = torch.Generator().manual_seed(1)
    res = {}
    for dtype in (torch.float64, torch.float32):
        x = feats.to(dtype).requires_grad_(True)
        out = decoder_layout_torch(x, grid.to(dtype), 2, 12, -2.1792, -4.2, 0.03125)
        if not res:
            ups = [torch.randn(o.shape, generator=g) for o in out]
        torch.autograd.backward(out, [u.to(dtype) for u in ups])
        res[dtype] = ([o.detach().numpy() for o in out], x.grad.numpy())
    ref, gref = C.decoder64(feats, grid, 2, 12, -2.1792, -4.2, 0.03125, [u.numpy() for u in ups])
    for i, r in enumerate(ref):
        _pin64(res[torch.float64][0][i], r, f"out {i}")
        _compare(res[torch.float32][0][i], r, ctx=f"fp32 out {i}")
    _pin64(res[torch.float64][1], gref, "grad")
    print(f"\n  decoder grad: fp32 restatement worst err/bound {_compare(res[torch.float32][1], gref, ctx='grad'):.3g}")
    _tightness("centers", ref[0])
    _tightness("grad", gref)


def test_loss_chain_bound_follows_the_tree():
    """The chain part of the sum's bound: thread t adds elements t, t + T, ... in order; K * sum of |running sums|."""
    t = np.arange(1, 11, dtype=f64)
    b = C.chain_bound(t, 4)           # threads 0..3: (1,5,9), (2,6,10), (3,7), (4,8)
    assert np.allclose(b / K, [1 + 6 + 15, 2 + 8 + 18, 3 + 10, 4 + 12])


# ---------------------------------------------------------------------------------------------- GPU: the epilogue

def _run_epilogue(color, allmap, rays, vms, depth_ratio, ups, dev, single=False):
    """The kernels on V stacked views (srf_views_*, camera records) or, `single`, one view through srf_epilogue_*."""
    from lara_b200.epilogue import (epilogue_backward_raw, epilogue_forward_raw, epilogue_views_backward_raw,
                                    epilogue_views_forward_raw)
    t = lambda a: None if a is None else torch.as_tensor(np.ascontiguousarray(a)).float().to(dev)    # noqa: E731
    V, _, H, W = color.shape
    c, a, r = t(color), t(allmap), t(rays)
    new = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)    # noqa: E731
    if single:
        o = [new(3, H, W), new(1, H, W), new(H, W), new(3, H, W), new(3, H, W), new(H, W)]
        vm = t(vms[0]).reshape(4, 4)
        epilogue_forward_raw(c[0], a[0], None if r is None else r[0], vm, depth_ratio, *o)
        g = [t(ups[k]) for k in OUT_KEYS]
        dc, da = epilogue_backward_raw(c[0], a[0], None if r is None else r[0], vm, depth_ratio, *g)
        o = [x[None] for x in o]
        dc, da = dc[None], da[None]
    else:
        cams = torch.zeros((V, 24), dtype=torch.float32)
        cams[:, :16] = torch.as_tensor(np.stack(vms)).reshape(V, 16)
        cams = cams.to(dev)
        o = [new(V, 3, H, W), new(V, 1, H, W), new(V, H, W), new(V, 3, H, W), new(V, 3, H, W), new(V, H, W)]
        epilogue_views_forward_raw(c, a, r, cams, depth_ratio, *o)
        g = [t(ups[k]) for k in OUT_KEYS]
        dc, da = epilogue_views_backward_raw(c, a, r, cams, depth_ratio, *g)
    torch.cuda.synchronize()
    outs = {k: x.cpu().numpy().reshape((V,) + ((3, H, W) if x.shape[1:2] == (3,) and x.ndim == 4 else (H, W)))
            for k, x in zip(OUT_KEYS, o)}
    return outs, dc.cpu().numpy(), da.cpu().numpy()


def _check_epilogue(color, allmap, rays, vms, depth_ratio, ups, dev, ctx, single=False, max_band=0):
    """Every output and gradient element of every view within its bound; band elements aside, whose number is at most
    `max_band`; infinite-bound elements checked for their properties: finite wherever the fp32 torch restatement is,
    and a pseudo normal of length 0 or alpha.  Returns (worst, band, infinite)."""
    V = color.shape[0]
    outs, dc, da = _run_epilogue(color, allmap, rays, vms, depth_ratio, ups, dev, single)
    worst, nband, ninf, ninf_grad = 0.0, 0, 0, 0
    for v in range(V):
        up_v = {k: (None if x is None else x[v]) for k, x in ups.items()}
        st = C.EpilogueState(color[v], allmap[v], None if rays is None else rays[v], vms[v], depth_ratio)
        ref, band, inf = C.epilogue64(None, None, None, None, None, state=st)
        rc, ra, excl = _vjp(st, up_v)
        for k in OUT_KEYS:
            worst = max(worst, _compare(outs[k][v], ref[k], band if k == "depth_normal" else None, f"{ctx} view {v} {k}"))
        worst = max(worst, _compare(dc[v], rc, None, f"{ctx} view {v} d_color"))
        worst = max(worst, _compare(da[v], ra, excl, f"{ctx} view {v} d_allmap"))
        assert (da[v][7] == 0).all()
        ninf_g = int((~np.isfinite(ra.e)).any(0).sum())
        if rays is None:
            assert not inf.any() and ninf_g == 0
        elif inf.any() or ninf_g:
            # no bound: every output and gradient is finite wherever LaRa's fp32 ops give a finite one (a -inf median
            # at depth_ratio = 1 puts a point at infinity, and torch's values are NaN there too) ...
            o32, gc32, ga32 = _torch_epilogue(color[v], allmap[v], rays[v], vms[v], depth_ratio, up_v, torch.float32)
            for k in OUT_KEYS:
                got = outs[k][v]
                assert np.isfinite(got[np.isfinite(o32[k].reshape(got.shape))]).all(), f"{ctx} view {v}: non-finite {k}"
            assert np.isfinite(dc[v][np.isfinite(gc32)]).all(), f"{ctx} view {v}: non-finite d_color"
            assert np.isfinite(da[v][np.isfinite(ga32)]).all(), f"{ctx} view {v}: non-finite d_allmap"
            # ... and the pseudo normal is 0 or of length alpha
            m = inf & np.isfinite(o32["depth_normal"]).all(0)
            dn = outs["depth_normal"][v][:, m]
            length, al = np.linalg.norm(dn.astype(f64), axis=0), allmap[v][1][m].astype(f64)
            assert np.isfinite(dn).all(), f"{ctx}: non-finite pseudo normal"
            assert ((length == 0) | (np.abs(length - al) <= 1e-5 * al)).all(), f"{ctx}: pseudo normal of wrong length"
        nband += int(band.sum())
        ninf += int(inf.sum())
        ninf_grad += ninf_g
    assert nband <= max_band, f"{ctx}: {nband} band pixels"
    print(f"  {ctx}: worst err/bound {worst:.3g}; band {nband}, infinite-bound pseudo normals {ninf}, infinite-bound "
          f"gradient pixels {ninf_grad}")
    return worst, nband, ninf


def _render_views(sc, cams, dev, raw=False):
    from lara_b200 import rasterizer as R
    from lara_b200 import scene as S
    settings = [S.settings_for(c, torch.ones(3), sc["sh_degree"], dev, R.GaussianRasterizationSettings) for c in cams]
    camt = R.pack_cameras(settings, dev)
    t = {k: sc[k].to(dev).contiguous() for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    H, W = cams[0].image_height, cams[0].image_width
    color, allmap, _, _ = R.forward_views_raw(t["means3D"], t["shs"], None, t["opacities"], t["scales"], t["rotations"],
                                              None, camt, cams[0].tanfovx, cams[0].tanfovy, H, W, sc["sh_degree"])
    return color.cpu().numpy(), allmap.cpu().numpy()


@pytest.fixture(scope="module")
def rendered():
    """Three distinct views of a cube of Gaussians with LaRa's rays: the silhouette leaves alpha == 0 background."""
    from lara_b200 import scene as S
    sc = S.scene(30000, 41)
    cams = S.cameras(3, 120, 150, 41)
    color, allmap = _render_views(sc, cams, torch.device("cuda:0"))
    rays = np.stack([lara_rays(c).numpy() for c in cams])
    vms = [c.viewmatrix.numpy().reshape(16) for c in cams]
    return color, allmap, rays, vms


@pytest.mark.gpu
@pytest.mark.parametrize("only", list(OUT_KEYS) + [None])
@pytest.mark.parametrize("depth_ratio", [0.0, 0.5])
def test_epilogue_on_renderings(cuda_device, rendered, only, depth_ratio):
    color, allmap, rays, vms = rendered
    V, _, H, W = color.shape
    assert (allmap[:, 1] == 0).mean() > 0.1 and (allmap[:, 1] > 0).mean() > 0.1
    ups = {k: (None if x is None else np.stack([x] * V)) for k, x in upstreams(H, W, 7, only).items()}
    ups = {k: (None if x is None else x * (1 + np.arange(V)).reshape((V,) + (1,) * (x.ndim - 1)).astype(np.float32))
           for k, x in ups.items()}
    worst, _, _ = _check_epilogue(color, allmap, rays, vms, depth_ratio, ups, cuda_device, f"renderings only={only}")
    assert worst < 1.0


SHAPES = [(37, 45), (64, 70), (9, 33), (1, 5), (2, 7), (3, 3), (3, 40), (40, 3), (5, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", SHAPES)
@pytest.mark.parametrize("depth_ratio", [0.0, 0.5, 1.0])
def test_epilogue_on_synthetic_edges(cuda_device, H, W, depth_ratio):
    """Silhouettes, one-pixel rows and columns, isolated pixels, colour at and beyond 0 and 1, overflowing D / alpha,
    NaN and +-inf medians; the single-view entry and the views entry (V = 3 distinct maps and cameras)."""
    cases = [synthetic(H, W, 100 + 10 * v + H + W, overflow=v > 0, bad_median=v > 1) for v in range(3)]
    color, allmap, rays = (np.stack([c[i] for c in cases]) for i in range(3))
    vms = [c[3] for c in cases]
    ups = {k: (None if x is None else np.stack([x] * 3)) for k, x in upstreams(H, W, 9).items()}
    _check_epilogue(color, allmap, rays, vms, depth_ratio, ups, cuda_device, f"synthetic {H}x{W} r={depth_ratio}",
                    max_band=3)
    one = {k: (None if x is None else x[:1]) for k, x in ups.items()}
    _check_epilogue(color[:1], allmap[:1], rays[:1], vms[:1], depth_ratio, one, cuda_device, "single view", single=True,
                    max_band=1)


@pytest.mark.gpu
def test_epilogue_without_rays(cuda_device, rendered):
    color, allmap, _, vms = rendered
    V, _, H, W = color.shape
    ups = {k: (None if x is None else np.stack([x] * V)) for k, x in upstreams(H, W, 11).items()}
    _check_epilogue(color, allmap, None, vms, 0.0, ups, cuda_device, "rays=None")
    _check_epilogue(color[:1], allmap[:1], None, vms[:1], 0.0, {k: (None if x is None else x[:1]) for k, x in ups.items()},
                    cuda_device, "rays=None single", single=True)


# -------------------------------------------------------------------------------------------------- GPU: the loss

def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _check_loss(planar, tar, it, B, prex, det, dev, up=3.0):
    from lara_b200.loss import scene_loss
    V, _, H, W = planar["image"].shape
    leaves = {k: v.to(dev).clone().requires_grad_(True) for k, v in planar.items()}
    out = {k + prex: (v.permute(0, 2, 3, 1) if v.ndim == 4 else v) for k, v in leaves.items()}
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        loss, stats = scene_loss(out, tar.to(dev), it, batch_scenes=B, prex=prex)
        (loss * up).backward()
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev)
    with_reg = it > 1000 and prex != "_fine"
    n = V * H * W
    blocks = min(1024, -(-n // 256)) if det else min(8 * _sm_count(), -(-n // 256))
    vals, grads = C.loss64(planar["image"], tar, planar["rend_normal"], planar["depth_normal"], planar["acc_map"],
                           planar["rend_dist"], with_reg, B, up, blocks)
    worst = 0.0
    for k, got in (("loss", float(loss)), ("mse", float(stats["mse" + prex]))) + \
            ((("distortion", float(stats["distortion"])), ("normal", float(stats["normal"]))) if with_reg else ()):
        v, e = vals[k]
        assert abs(got - v) <= e, (k, got, v, e)
        worst = max(worst, abs(got - v) / e if e > 0 else 0.0)
    for k, g in grads.items():
        if g is None:
            assert leaves[k].grad is None or float(leaves[k].grad.abs().max()) == 0.0, k
            continue
        worst = max(worst, _compare(leaves[k].grad.cpu().numpy(), g, ctx=f"loss {k}"))
    print(f"  loss V={V} {H}x{W} iter={it} B={B} prex={prex!r} det={det}: worst err/bound {worst:.3g}, sum bound / sum "
          f"{vals['sums'][1][0] / vals['sums'][0][0]:.3g}")
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("V,H,W,it,B,prex,det", [
    (3, 37, 45, 1000, 1, "", False), (3, 37, 45, 1001, 2, "", False), (3, 37, 45, 1001, 2, "", True),
    (2, 50, 72, 5000, 1, "_fine", False), (8, 512, 512, 5000, 1, "", False), (8, 512, 512, 5000, 3, "", True)])
def test_loss_per_element(cuda_device, V, H, W, it, B, prex, det):
    planar, tar = _loss_case(V, H, W, V + H + it)
    planar = {k: (v * 2.0 - 0.5 if k == "image" else v) for k, v in planar.items()}     # beyond [0, 1] too
    assert (V * H * W) % 256 != 0 or V * H * W > 8 * 132 * 256
    _check_loss(planar, tar, it, B, prex, det, cuda_device)


# ----------------------------------------------------------------------------------------------- GPU: the decoder

@pytest.mark.gpu
@pytest.mark.parametrize("B,N,K_,sh_dim", [(1, 1000, 2, 12), (3, 4097, 1, 12), (2, 515, 2, 48), (1, 200, 3, 3)])
def test_decoder_per_element(cuda_device, B, N, K_, sh_dim):
    from lara_b200.decoder_layout import gaussians_from_decoder
    feats, grid = _decoder_case(B, N, K_, sh_dim, N)
    x = feats.to(cuda_device).requires_grad_(True)
    out = gaussians_from_decoder(x, grid.to(cuda_device), K_, sh_dim, -2.1792, -4.2, 0.03125)
    g = torch.Generator().manual_seed(N + 1)
    ups = [torch.randn(o.shape, generator=g) for o in out]
    torch.autograd.backward(out, [u.to(cuda_device) for u in ups])
    ref, gref = C.decoder64(feats, grid, K_, sh_dim, -2.1792, -4.2, 0.03125, [u.numpy() for u in ups])
    worst = max(_compare(o.detach().cpu().numpy(), r, ctx=f"decoder out {i}") for i, (o, r) in enumerate(zip(out, ref)))
    worst = max(worst, _compare(x.grad.cpu().numpy(), gref, ctx="decoder grad"))
    print(f"  decoder B={B} N={N} K={K_} sh_dim={sh_dim}: worst err/bound {worst:.3g}")


# -------------------------------------------------------------------------------------- GPU: the chain, link by link

def _chain(dev, det, ms_ssim, fine=False):
    """decoder output -> gaussians_from_decoder -> render_scene_views (raw activations, LaRa rays, V = 3) ->
    scene_loss(iter=5000) -> backward, with every boundary's maps kept.  `fine`: LaRa's fine pass as well -- a seeded
    mask with voxels of 0, 1 and 2 masked Gaussians, sample_point_feats on the first n_sel = 2 coarse views,
    FineHead(80, 12).fine_shs on a volume_feat_up leaf, the masked render and scene_loss(prex="_fine") added to the
    coarse loss."""
    from lara_b200 import rasterizer as R
    from lara_b200 import scene as S
    from lara_b200.decoder_layout import gaussians_from_decoder
    from lara_b200.loss import scene_loss
    from lara_b200.multiview import render_scene_views
    B, N, K_, sh_dim = 1, 9000, 2, 12
    H, W, V = 168, 144, 3
    g = torch.Generator().manual_seed(77)
    C_ = 10 + sh_dim
    feats = torch.randn((B, N, K_ * C_), generator=g)
    feats.view(B, N, K_, C_)[..., 3:3 + sh_dim] *= 0.5
    feats.view(B, N, K_, C_)[..., 3 + sh_dim] = feats.view(B, N, K_, C_)[..., 3 + sh_dim] * 1.5 + 1.0
    feats.view(B, N, K_, C_)[..., 4 + sh_dim:6 + sh_dim] *= 0.3
    grid = (torch.rand((N, 3), generator=g) - 0.5) * 0.9
    cams = S.cameras(V, H, W, 77)
    rays = torch.stack([lara_rays(c) for c in cams]).to(dev)
    settings = [S.settings_for(c, torch.ones(3), 1, dev, R.GaussianRasterizationSettings) for c in cams]
    tar = torch.rand((V, H, W, 3), generator=g).to(dev)
    x = feats.to(dev).requires_grad_(True)
    if ms_ssim:
        # against uniform noise cs is about 0, so relu would leave the MS-SSIM term without a gradient or with
        # planes whose sign is undecided: a target correlated with a first rendering instead
        from test_ms_ssim import smooth_pair
        with torch.no_grad():
            dec = gaussians_from_decoder(x, grid.to(dev), K_, sh_dim, -2.1792, -4.2, 0.5 / 16)
            centers, shs, scaling, rotation, opacity = (t.reshape((-1,) + tuple(t.shape[2:])) for t in dec)
            img = render_scene_views(centers, shs, opacity, scaling, rotation, settings, rays=rays,
                                     raw_activations=True)["image"]
        _, pert = smooth_pair(V, 3, H, W, 78, dtype=torch.float32)
        tar = (img + 0.1 * (pert.to(dev).permute(0, 2, 3, 1) - 0.5)).clamp(0, 1).contiguous()
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        dec = gaussians_from_decoder(x, grid.to(dev), K_, sh_dim, -2.1792, -4.2, 0.5 / 16)
        for t in dec:
            t.retain_grad()
        centers, shs, scaling, rotation, opacity = (t.reshape((-1,) + tuple(t.shape[2:])) for t in dec)
        out = render_scene_views(centers, shs, opacity, scaling, rotation, settings, rays=rays, raw_activations=True)
        for k in OUT_KEYS:
            out[k].retain_grad()
        loss, stats = scene_loss(out, tar, 5000, ms_ssim=ms_ssim)
        extra = _fine_pass(dev, out, centers, shs, opacity, scaling, rotation, cams, settings, rays, tar, N, K_,
                           sh_dim) if fine else {}
        total = loss + extra["loss_fine"] if fine else loss
        (total * 2.0).backward()
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev)
    return dict(feats=feats, grid=grid, x=x, dec=dec, out=out, loss=loss, stats=stats, tar=tar, cams=cams, rays=rays,
                settings=settings, params=(centers, shs, opacity, scaling, rotation), K=K_, sh_dim=sh_dim, **extra)


N_SEL = 2


def _pinhole(cams):
    """w2c [V,4,4] and the pinhole ixt [V,3,3] of the cameras (principal point at the image centre)."""
    w2c = torch.stack([c.viewmatrix.T for c in cams]).contiguous()
    ixt = torch.zeros((len(cams), 3, 3))
    for v, c in enumerate(cams):
        W, H = c.image_width, c.image_height
        ixt[v, 0, 0], ixt[v, 1, 1] = W / (2 * c.tanfovx), H / (2 * c.tanfovy)
        ixt[v, 0, 2], ixt[v, 1, 2], ixt[v, 2, 2] = W / 2, H / 2, 1.0
    return w2c, ixt


def _fine_pass(dev, out, centers, shs, opacity, scaling, rotation, cams, settings, rays, tar, N, K_, sh_dim):
    from lara_b200.loss import scene_loss
    from lara_b200.multiview import render_scene_views
    from lara_b200.point_feats import sample_point_feats
    from test_fine_head import _head
    V, H, W = len(cams), cams[0].image_height, cams[0].image_width
    g = torch.Generator().manual_seed(79)
    mask = (torch.rand((N * K_,), generator=g) < 0.5).to(dev)
    per_voxel = mask.view(N, K_).sum(1)
    assert all(bool((per_voxel == c).any()) for c in range(K_ + 1))
    img_ref = torch.rand((N_SEL, 3, H, W), generator=g).to(dev)
    vf = (torch.randn((N, 80), generator=g) * 0.5 + 0.3).to(dev).requires_grad_(True)
    head = _head(80, sh_dim, 13, dev)
    w2c, ixt = (t.to(dev) for t in _pinhole(cams))
    pts = centers[mask]
    pts.retain_grad()
    pf = sample_point_feats(pts, img_ref, {k: out[k][:N_SEL] for k in ("image", "acc_map", "depth")}, w2c[:N_SEL],
                            ixt[:N_SEL])
    pf.retain_grad()
    shs_fine = head.fine_shs(vf, K_, mask, pf, shs)
    fp = [centers[mask], shs_fine, opacity[mask], scaling[mask], rotation[mask]]
    for t in fp:
        t.retain_grad()
    fine = render_scene_views(fp[0], fp[1], fp[2], fp[3], fp[4], settings, rays=rays, raw_activations=True,
                              prex="_fine")
    for k in OUT_KEYS:
        fine[k + "_fine"].retain_grad()
    loss_fine, _ = scene_loss(fine, tar, 5000, prex="_fine")
    return dict(mask=mask, img_ref=img_ref, vf=vf, head=head, w2c=w2c, ixt=ixt, pts=pts, pf=pf, fine_params=fp,
                fine=fine, loss_fine=loss_fine)


def _render_link(prm, camt, cams, rays, dev):
    """The renderer's forward again on the node's parameters (deterministic, so its state is the node's) and the
    epilogue forward on its maps.  Returns (color, allmap, radii, state, [six epilogue outputs])."""
    from lara_b200 import rasterizer as R
    from lara_b200.epilogue import epilogue_views_forward_raw
    centers, shs, opacity, scaling, rotation = prm
    V, H, W = len(cams), cams[0].image_height, cams[0].image_width
    color, allmap, radii, state = R.forward_views_raw(centers, shs, None, opacity, scaling, rotation, None, camt,
                                                      cams[0].tanfovx, cams[0].tanfovy, H, W, 1, raw_activations=True)
    new = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)     # noqa: E731
    o = [new(V, 3, H, W), new(V, 1, H, W), new(V, H, W), new(V, 3, H, W), new(V, 3, H, W), new(V, H, W)]
    epilogue_views_forward_raw(color, allmap, rays, camt, 0.0, *o)
    return color, allmap, radii, state, o


def _node_planar(out, prex=""):
    """The node's six outputs and their gradients, planar."""
    pl = lambda t: None if t is None else (t.permute(0, 3, 1, 2) if t.ndim == 4 else t).contiguous()    # noqa: E731
    return ({k: pl(out[k + prex].detach()) for k in OUT_KEYS}, {k: pl(out[k + prex].grad) for k in OUT_KEYS})


def _epilogue_fwd_link(o, out_nodes, col, am, rays, vms, ctx):
    """The re-run epilogue equals the node bit for bit, and every view's outputs lie within epilogue64's bound."""
    for k, t in zip(OUT_KEYS, o):
        assert torch.equal(t, out_nodes[k]), f"{ctx} {k}"
    w = 0.0
    for v in range(col.shape[0]):
        st = C.EpilogueState(col[v], am[v], rays[v], vms[v], 0.0)
        r, band, _ = C.epilogue64(None, None, None, None, None, state=st)
        assert band.sum() == 0
        for k, t in zip(OUT_KEYS, o):
            w = max(w, _compare(t[v].cpu().numpy(), r[k], ctx=f"{ctx} epilogue fwd view {v} {k}"))
    return w


def _epilogue_vjp_link(color, allmap, rays_t, camt, col, am, rays, vms, gpl, ctx):
    """The epilogue backward given the node's upstream maps, every element within epilogue_vjp64's bound.  Returns
    (d_color, d_allmap, worst)."""
    from lara_b200.epilogue import epilogue_views_backward_raw
    d_color, d_allmap = epilogue_views_backward_raw(color, allmap, rays_t, camt, 0.0, gpl["image"], gpl["depth"],
                                                    gpl["acc_map"], gpl["rend_normal"], gpl["depth_normal"],
                                                    gpl["rend_dist"])
    dc, da = d_color.cpu().numpy(), d_allmap.cpu().numpy()
    w = 0.0
    for v in range(col.shape[0]):
        st = C.EpilogueState(col[v], am[v], rays[v], vms[v], 0.0)
        up = {k: (None if g is None else g[v].cpu().numpy()) for k, g in gpl.items()}
        rc, ra, excl = _vjp(st, up)
        assert excl.sum() == 0
        w = max(w, _compare(dc[v], rc, ctx=f"{ctx} epilogue vjp view {v} d_color"),
                _compare(da[v], ra, ctx=f"{ctx} view {v} d_allmap"))
    return d_color, d_allmap, w


GAUSS_KEYS = ("means3D", "sh", "opacities", "scales", "rotations")


def _replay_link(state, radii, prm, camt, cams, d_color, d_allmap, det, ctx):
    """The per-Gaussian backward given d_color / d_allmap, against the float64 replay of every view.  Returns
    (kernel gradients, replay {key: (value, bound)}, band mask, worst)."""
    from lara_b200 import rasterizer as R
    from lara_b200.debug import unpack_state
    from oracle import oracle as O
    from test_grad_per_gaussian import _cam_dict
    centers, shs, opacity, scaling, rotation = prm
    V, H, W = len(cams), cams[0].image_height, cams[0].image_width
    P = centers.shape[0]
    g = R.backward_views_raw(state, radii, centers, shs, None, scaling, rotation, None, camt, cams[0].tanfovx,
                             cams[0].tanfovy, H, W, 1, d_color, d_allmap, raw_activations=True, deterministic=det)
    torch.cuda.synchronize()
    dc, da = d_color.cpu().numpy(), d_allmap.cpu().numpy()
    p = dict(means3D=centers.cpu().numpy(), shs=shs.cpu().numpy(), sh_degree=1, opacities=opacity.cpu().numpy(),
             scales=scaling.cpu().numpy(), rotations=rotation.cpu().numpy(), raw_activations=True)
    views, band = [], np.zeros(P, bool)
    for v in range(V):
        u = {k: x.cpu().numpy() for k, x in unpack_state(state, P, H, W, view=v).items()}
        u["visible"] = radii[v].cpu().numpy() > 0
        r = O.replay(u, np.ones(3, np.float32), dc[v], da[v])
        views.append(O.view_vjp(u, r["g"], r["g_e"], p, _cam_dict(cams[v])))
        band |= r["band"] != 0
    ref = O.gaussian_grads(views, p, u["opacity"])
    assert band.sum() < 1e-4 * P + 1, f"{ctx}: {int(band.sum())} band Gaussians"
    w = 0.0
    for k in GAUSS_KEYS:
        v_, e_ = ref[k]
        w = max(w, _compare(g[k].cpu().numpy().reshape(v_.shape), EB(v_, e_), _band(band, v_), f"{ctx} per-Gaussian {k}"))
    return g, ref, band, w


def _band(band, v_):
    return band.reshape((-1,) + (1,) * (v_.ndim - 1))


@pytest.mark.gpu
@pytest.mark.parametrize("det,ms_ssim", [(False, False), (True, False), (False, True)])
def test_lara_chain_link_by_link(cuda_device, det, ms_ssim):
    from lara_b200 import rasterizer as R
    dev = cuda_device
    ch = _chain(dev, det, ms_ssim)
    cams, settings, out = ch["cams"], ch["settings"], ch["out"]
    V, H, W = len(cams), cams[0].image_height, cams[0].image_width
    prm = tuple(t.detach().contiguous() for t in ch["params"])
    camt = R.pack_cameras(settings, dev)
    # the node's state, repeated: the forward is deterministic, so its epilogue outputs equal the node's bit for bit
    color, allmap, radii, state, o = _render_link(prm, camt, cams, ch["rays"], dev)
    nodes, gpl = _node_planar(out)
    col, am, rays = color.cpu().numpy(), allmap.cpu().numpy(), ch["rays"].cpu().numpy()
    vms = [c.viewmatrix.numpy().reshape(16) for c in cams]
    worst = {}
    # 1. decoder forward
    ref, _ = C.decoder64(ch["feats"], ch["grid"], ch["K"], ch["sh_dim"], -2.1792, -4.2, 0.5 / 16)
    worst["decoder fwd"] = max(_compare(t.detach().cpu().numpy(), r, ctx="decoder fwd") for t, r in zip(ch["dec"], ref))
    # 2. epilogue forward and 3. the loss, given their actual fp32 inputs
    worst["epilogue fwd"] = _epilogue_fwd_link(o, nodes, col, am, rays, vms, "coarse")
    pl = {k: t.cpu() for k, t in zip(OUT_KEYS, o)}
    n = V * H * W
    blocks = min(1024, -(-n // 256)) if det else min(8 * _sm_count(), -(-n // 256))
    vals, lg = C.loss64(pl["image"], ch["tar"].cpu(), pl["rend_normal"], pl["depth_normal"], pl["acc_map"],
                        pl["rend_dist"], True, 1, 2.0, blocks)
    loss_ref = EB(*vals["loss"])
    w = 0.0
    if ms_ssim:
        # + (0.5 / B) (1 - s) in fp32 torch ops; the MS-SSIM gradient for autograd's upstream fp32(-0.5 * 2.0) on the
        # views side by side, added to the MSE gradient in fp32
        from oracle import ms_ssim64 as M
        cat = lambda a: np.concatenate(list(a), axis=-1)[None]          # noqa: E731
        ms = M.ms_ssim64(cat(pl["image"].numpy()), cat(ch["tar"].cpu().permute(0, 3, 1, 2).numpy()), 1.0, True,
                         [float(np.float32(-0.5 * 2.0))])
        assert all(p["state"] == "pos" for p in ms["planes"].values()), [p["m"] for p in ms["planes"].values()]
        s = EB(*ms["out"][0])
        w = max(w, _compare(float(ch["stats"]["ssim"]), s, ctx="ssim stat"))
        loss_ref = M.Bound.add(loss_ref, M.Bound.scale(M.Bound.sub(1.0, s), 0.5))
        gv = np.stack([ms["planes"][(0, c)]["dX"][0].v for c in range(3)]).reshape(3, H, V, W).transpose(2, 0, 1, 3)
        ge = np.stack([ms["planes"][(0, c)]["dX"][0].e for c in range(3)]).reshape(3, H, V, W).transpose(2, 0, 1, 3)
        lg["image"] = M.Bound.add(lg["image"], EB(gv, ge))
    w = max(w, _compare(float(ch["loss"].detach()), loss_ref, ctx="loss value"))
    worst["loss"] = max([w] + [_compare(gpl[k].cpu().numpy(), g, ctx=f"loss {k}") for k, g in lg.items()])
    if ms_ssim:
        worst["loss value, ssim stat and g_image with MS-SSIM"] = max(w, _compare(gpl["image"].cpu().numpy(), lg["image"]))
    assert gpl["depth"] is None and gpl["acc_map"] is None
    # 4. epilogue vjp, given the node's upstream maps
    d_color, d_allmap, worst["epilogue vjp"] = _epilogue_vjp_link(color, allmap, ch["rays"], camt, col, am, rays, vms,
                                                                  gpl, "coarse")
    # 5. per-Gaussian gradients: the replay of every view with the kernel's d_color / d_allmap
    g, ref, band, w = _replay_link(state, radii, prm, camt, cams, d_color, d_allmap, det, "coarse")
    node = {"means3D": ch["dec"][0].grad, "sh": ch["dec"][1].grad, "scales": ch["dec"][2].grad,
            "rotations": ch["dec"][3].grad, "opacities": ch["dec"][4].grad}
    for k in GAUSS_KEYS:
        v_, e_ = ref[k]
        if det:
            assert torch.equal(g[k].reshape(-1), node[k].reshape(-1)), k     # the decomposition is the node's
        w = max(w, _compare(node[k].cpu().numpy().reshape(v_.shape), EB(v_, e_), _band(band, v_), f"node {k}"))
    worst["per-Gaussian"] = w
    # 6. decoder backward, given the node's parameter gradients
    _, gref = C.decoder64(ch["feats"], ch["grid"], ch["K"], ch["sh_dim"], -2.1792, -4.2, 0.5 / 16,
                          [t.grad.cpu().numpy() for t in ch["dec"]])
    worst["decoder bwd"] = _compare(ch["x"].grad.cpu().numpy(), gref, ctx="decoder bwd")
    print(f"\n  chain det={det} ms_ssim={ms_ssim}: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()) +
          f"; band-excluded Gaussians {int(band.sum())}")


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True])
def test_lara_fine_chain_link_by_link(cuda_device, det):
    """The coarse chain with LaRa's fine pass, link by link on each link's actual fp32 inputs: the sampler against
    point_feats64, the head against fine_head_torch in float64 (1e-5 of each tensor's maximum), the fine render's
    epilogue, loss and per-Gaussian replay through the coarse chain's helpers, and where the passes meet: the coarse
    image / acc_map / depth node gradients (loss part + sampler part on views < n_sel), the Gaussians' node gradients
    (coarse + mask-scattered fine + sampler point part) with the head's residual into shs, then the decoder backward."""
    from lara_b200 import rasterizer as R
    from oracle import point_feats64 as P
    from oracle.fine_head_torch import fine_shs_torch
    from test_fine_head import TOL, _err
    from test_point_feats_per_element import _kernels
    dev = cuda_device
    ch = _chain(dev, det, False, fine=True)
    cams, settings, out, fine = ch["cams"], ch["settings"], ch["out"], ch["fine"]
    V, H, W = len(cams), cams[0].image_height, cams[0].image_width
    prm = tuple(t.detach().contiguous() for t in ch["params"])
    camt = R.pack_cameras(settings, dev)
    rays, rays_t = ch["rays"].cpu().numpy(), ch["rays"]
    vms = [c.viewmatrix.numpy().reshape(16) for c in cams]
    n = V * H * W
    blocks = min(1024, -(-n // 256)) if det else min(8 * _sm_count(), -(-n // 256))
    mask = ch["mask"]
    sfx = "_det" if det else ""
    worst = {}
    # coarse forward: render, epilogue and the loss value on their inputs
    color, allmap, radii, state, o = _render_link(prm, camt, cams, rays_t, dev)
    nodes, gpl = _node_planar(out)
    col, am = color.cpu().numpy(), allmap.cpu().numpy()
    worst["coarse epilogue fwd"] = _epilogue_fwd_link(o, nodes, col, am, rays, vms, "coarse")
    pl = {k: t.cpu() for k, t in zip(OUT_KEYS, o)}
    vals, lg = C.loss64(pl["image"], ch["tar"].cpu(), pl["rend_normal"], pl["depth_normal"], pl["acc_map"],
                        pl["rend_dist"], True, 1, 2.0, blocks)
    worst["coarse loss value"] = _compare(float(ch["loss"].detach()), EB(*vals["loss"]), ctx="coarse loss value")
    # the sampler on its actual inputs: forward and the node's vjp; its rendering gradients from a re-run
    pts = prm[0][mask]
    rend = {k: out[k][:N_SEL].detach() for k in ("image", "acc_map", "depth")}
    case = (pts, ch["img_ref"], rend, ch["w2c"][:N_SEL], ch["ixt"][:N_SEL])
    up = ch["pf"].grad
    st = P.point_feats64(pts, case[3], case[4], ch["img_ref"], rend["image"].permute(0, 3, 1, 2), rend["acc_map"],
                         rend["depth"][..., 0], up)
    assert not st["inf_pairs"].any()
    rerun = _kernels(case, up, det, dev)
    worst["sampler"] = max(_compare(ch["pf"].detach().cpu().numpy(), st["feats"], ctx="sampler feats"),
                           _compare(ch["pts"].grad.cpu().numpy(), st["g_points"], ctx="sampler g_points (node)"),
                           _compare(rerun["g_points"], st["g_points"], ctx="sampler g_points"),
                           *[_compare(rerun[k], st[k + sfx], ctx=f"sampler {k}") for k in ("g_image", "g_acc", "g_depth")])
    # the head against float64, on the node's inputs and upstream
    params = [p.detach().double() for p in ch["head"]._params()]
    vf64 = ch["vf"].detach().double().requires_grad_(True)
    pf64 = ch["pf"].detach().double().requires_grad_(True)
    shs64 = prm[1].double().requires_grad_(True)
    shs_fine = ch["fine_params"][1]
    o64 = fine_shs_torch(vf64, ch["K"], mask, pf64, shs64, params)
    o64.backward(shs_fine.grad.double())
    head = {"out": _err(shs_fine.detach(), o64.detach()), "g_volume_feat": _err(ch["vf"].grad, vf64.grad),
            "g_point_feats": _err(ch["pf"].grad, pf64.grad)}
    assert all(e <= TOL for e in head.values()), head
    # the fine render: epilogue, loss (no regularisers under prex="_fine") and per-Gaussian replay
    fprm = tuple(t.detach().contiguous() for t in ch["fine_params"])
    colorf, allmapf, radiif, statef, of = _render_link(fprm, camt, cams, rays_t, dev)
    nodesf, gplf = _node_planar(fine, "_fine")
    colf, amf = colorf.cpu().numpy(), allmapf.cpu().numpy()
    worst["fine epilogue fwd"] = _epilogue_fwd_link(of, nodesf, colf, amf, rays, vms, "fine")
    plf = {k: t.cpu() for k, t in zip(OUT_KEYS, of)}
    valsf, lgf = C.loss64(plf["image"], ch["tar"].cpu(), plf["rend_normal"], plf["depth_normal"], plf["acc_map"],
                          plf["rend_dist"], False, 1, 2.0, blocks)
    w = _compare(float(ch["loss_fine"].detach()), EB(*valsf["loss"]), ctx="fine loss value")
    worst["fine loss"] = max(w, _compare(gplf["image"].cpu().numpy(), lgf["image"], ctx="fine loss image"))
    assert all(gplf[k] is None or not bool(gplf[k].any()) for k in OUT_KEYS if k != "image")
    dcf, daf, worst["fine epilogue vjp"] = _epilogue_vjp_link(colorf, allmapf, rays_t, camt, colf, amf, rays, vms,
                                                              gplf, "fine")
    _, reff, bandf, worst["fine per-Gaussian"] = _replay_link(statef, radiif, fprm, camt, cams, dcf, daf, det, "fine")
    fnode = dict(zip(GAUSS_KEYS, (ch["fine_params"][0].grad, shs_fine.grad, ch["fine_params"][2].grad,
                                  ch["fine_params"][3].grad, ch["fine_params"][4].grad)))
    for k in GAUSS_KEYS:
        v_, e_ = reff[k]
        worst["fine per-Gaussian"] = max(worst["fine per-Gaussian"], _compare(
            fnode[k].cpu().numpy().reshape(v_.shape), EB(v_, e_), _band(bandf, v_), f"fine node {k}"))
    # where the passes meet (1): the coarse nodes' gradients, loss part + sampler part on the first n_sel views
    samp = {"image": st["g_image" + sfx], "acc_map": st["g_acc" + sfx], "depth": st["g_depth" + sfx]}
    w = 0.0
    for k in ("image", "acc_map", "depth"):
        shape = gpl[k].shape
        base = lg[k] if k == "image" else EB(np.zeros(shape))
        part = EB(np.zeros(shape), np.zeros(shape))
        part.v[:N_SEL] = samp[k].v.reshape((N_SEL,) + shape[1:])
        part.e[:N_SEL] = samp[k].e.reshape((N_SEL,) + shape[1:])
        w = max(w, _compare(gpl[k].cpu().numpy(), P.add(EB(base.v, base.e), part), ctx=f"coarse node {k}"))
    worst["coarse nodes: loss + sampler"] = w
    # the coarse epilogue vjp and replay, given those node gradients
    d_color, d_allmap, worst["coarse epilogue vjp"] = _epilogue_vjp_link(color, allmap, rays_t, camt, col, am, rays,
                                                                         vms, gpl, "coarse")
    _, ref, band, worst["coarse per-Gaussian"] = _replay_link(state, radii, prm, camt, cams, d_color, d_allmap, det,
                                                              "coarse")
    # where the passes meet (2): the Gaussians' node gradients, coarse + mask-scattered fine (+ the sampler's point
    # gradient into the means, the head's residual into shs), in any order of autograd's additions
    m = mask.cpu().numpy()
    node = {"means3D": ch["dec"][0].grad, "sh": ch["dec"][1].grad, "scales": ch["dec"][2].grad,
            "rotations": ch["dec"][3].grad, "opacities": ch["dec"][4].grad}
    w = 0.0
    for k in GAUSS_KEYS:
        v_, e_ = ref[k]
        fv, fe = np.zeros_like(v_), np.zeros_like(e_)
        fv[m], fe[m] = reff[k][0], reff[k][1]
        terms = [EB(v_, e_), EB(fv, fe)]
        if k == "means3D":
            sv, se = np.zeros_like(v_), np.zeros_like(e_)
            sv[m], se[m] = st["g_points"].v, st["g_points"].e
            terms.append(EB(sv, se))
        excl = _band(band, v_).copy()
        excl[m] |= _band(bandf, reff[k][0])
        w = max(w, _compare(node[k].cpu().numpy().reshape(v_.shape), P.sum_any_order(terms), excl, f"node {k}"))
    worst["Gaussian nodes: coarse + fine + sampler"] = w
    # the decoder backward, given the node's parameter gradients
    _, gref = C.decoder64(ch["feats"], ch["grid"], ch["K"], ch["sh_dim"], -2.1792, -4.2, 0.5 / 16,
                          [t.grad.cpu().numpy() for t in ch["dec"]])
    worst["decoder bwd"] = _compare(ch["x"].grad.cpu().numpy(), gref, ctx="decoder bwd")
    print(f"\n  fine chain det={det}: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()) +
          f"; head (err / max) " + ", ".join(f"{k} {v:.2g}" for k, v in head.items()) +
          f"; masked Gaussians {int(m.sum())}, widened sampler pairs {int(st['wide_pairs'].sum())}, band-excluded "
          f"Gaussians {int(band.sum())} coarse, {int(bandf.sum())} fine")
    _tightness("sampler g_points", st["g_points"])
