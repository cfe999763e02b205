"""The fine pass's point-feature sampler (csrc/point_feats.cu) element by element against float64.

``oracle.point_feats64`` restates the kernels' formulas in float64 with a bound per element on what their fp32
evaluation may differ by (its docstring derives the rules).  So a pixel reached only by a tap of weight 2^-20, a border
pixel one or two taps reach, a point far from the camera with a small gradient and a pixel that sums 10^5 terms are
each held to their own bound, not to a fraction of the tensor's largest element.  Where a decision of the kernels --
``floor(ix)``, ``floor(iy)`` (and with them the border taps' in/out tests) or ``sign(s_depth - z)`` -- is not decided
by the bound, the element is checked against the hull of every side, and the number of such elements is printed.

CPU part: the statement equals the plain-torch restatement run in float64; the fp32 restatement and an fp32 NumPy
emulation of the kernels' operation sequence (both summation modes) lie within the bound at every element; the host
restatement of det_sum.cuh equals det_sum.cuh compiled for the host.  GPU part: the kernels, with the default backward
and with ``torch.use_deterministic_algorithms(True)``.

The pile-up case bites in deterministic mode only: with atomics in an unknown order, the default path's order-free
bound on a pixel of 66 667 random-signed terms is about as large as the value itself, so a default-mode pass there
would not notice a few hundred dropped terms; det_sum's fixed-point bound is about 400 times tighter.
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import point_feats64 as P
from oracle.oracle import EB
from test_chain_per_element import _pin64, _tightness
from test_deterministic import _sum as _host_sum
from test_deterministic import host  # noqa: F401  (det_sum.cuh compiled for the host: a fixture)
from test_point_feats import make_case, point_feats_torch

f32, f64 = np.float32, np.float64


# ------------------------------------------------------------------------------------------------------------- checks

def _check(got, ref: EB, ctx, excl=None):
    """|got - ref| <= bound at every element (outside `excl`); the worst err/bound."""
    a = np.asarray(got, f64).reshape(ref.v.shape)
    err = np.abs(a - ref.v)
    keep = np.ones(ref.v.shape, bool) if excl is None else ~np.broadcast_to(excl, ref.v.shape)
    bad = ~(err <= ref.e) & keep
    if bad.any():
        i = tuple(int(j) for j in np.argwhere(bad)[0])
        raise AssertionError(f"{ctx}: {int(bad.sum())} of {bad.size} elements outside their bound, first at {i}: "
                             f"got {a[i]!r}, float64 {ref.v[i]!r}, bound {ref.e[i]!r}")
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(keep & (err > 0), err / ref.e, 0.0)
    return float(r.max()) if r.size else 0.0


def _planar(rend):
    """image [V,H,W,3] -> [V,3,H,W], depth [V,H,W,1] -> [V,H,W]."""
    f = lambda t: t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)       # noqa: E731
    return f(rend["image"]).transpose(0, 3, 1, 2), f(rend["acc_map"]), f(rend["depth"])[..., 0]


def statement(case, up):
    points, img_ref, rend, w2c, ixt = case
    image, acc, depth = _planar(rend)
    return P.point_feats64(points, w2c, ixt, img_ref, image, acc, depth, up)


def check_all(res, st, det, ctx):
    """Every output element of `res` (feats, g_points, g_image, g_acc, g_depth as arrays) within the statement's
    bound; prints the worst err/bound, the tightness and the widened counts.  Returns the worst."""
    sfx = "_det" if det else ""
    assert not st["inf_pairs"].any(), f"{ctx}: {int(st['inf_pairs'].sum())} pairs with an infinite bound"
    wp, wx = st["wide_pairs"][:, None, :], st["wide_pixels"]
    excl = {"feats": wp, "g_points": st["wide_points"][:, None], "g_image": wx[:, :3], "g_acc": wx[:, 3], "g_depth": wx[:, 4]}
    w, dec = {}, {}
    for k in excl:
        ref = st[k + (sfx if k.startswith("g_") and k != "g_points" else "")]
        w[k] = _check(res[k], ref, f"{ctx} {k}")
        dec[k] = _check(res[k], ref, f"{ctx} {k}", excl[k])
    # a widened element may sit at its hull's end (the kernel took one side): its err/bound approaches 1
    print(f"\n  {ctx}: worst err/bound " + ", ".join(f"{k} {v:.3g}" for k, v in w.items()) +
          "; outside the widened elements " + ", ".join(f"{k} {v:.3g}" for k, v in dec.items()) +
          f"; widened pairs {int(st['wide_pairs'].sum())}, point-gradient elements {3 * int(st['wide_points'].sum())}"
          f", rendering-gradient elements {int(st['wide_pixels'].sum())}; most terms in one pixel {st['max_terms']}")
    for k in ("feats", "g_points", "g_image", "g_depth"):
        _tightness(k, st[k + (sfx if k in ("g_image", "g_depth") else "")])
    return max(w.values())


# ------------------------------------------------------------------------------------------- fp32 emulation (NumPy)

def _fma(a, b, c):
    """fmaf as one float64 operation rounded to fp32."""
    return (np.asarray(a, f64) * np.asarray(b, f64) + np.asarray(c, f64)).astype(f32)


def _coord(xs, size):
    s = f32(size)
    g = ((xs + f32(0.5)) / s) * f32(2.0) - f32(1.0)
    return ((g + f32(1.0)) * s - f32(1.0)) / f32(2.0)


def emulate(points, w2c, ixt, img_ref, image, acc, depth, g_feats, det):
    """The kernels' operation sequence in fp32 (point_feats.cu), one thread per point, the atomics in point order."""
    pts, E_, K_ = (np.asarray(a, f32) for a in (points, w2c, ixt))
    V, _, H, W = img_ref.shape
    n, HW = pts.shape[0], H * W
    planes = np.concatenate([img_ref.reshape(V, 3, HW), image.reshape(V, 3, HW), acc.reshape(V, 1, HW),
                             depth.reshape(V, 1, HW)], 1).astype(f32)
    g = np.asarray(g_feats, f32)
    feats = np.zeros((V, 8, n), f32)
    gpt = np.zeros((n, 3), f32)
    rend = np.zeros((V, 5, HW), f32)
    fixed = np.zeros((V, 5, HW), np.int64)
    L = P.ceil_log2(4 * V * n)
    kq = P.scale_exp(P.abs_bits_max(g), L)
    x = [pts[:, k] for k in range(3)]
    with np.errstate(all="ignore"):
        for v in range(V):
            E, Km = E_[v], K_[v]
            q = [_fma(x[2], E[r, 2], _fma(x[1], E[r, 1], x[0] * E[r, 0])) + E[r, 3] for r in range(3)]
            p = [_fma(q[2], Km[r, 2], _fma(q[1], Km[r, 1], q[0] * Km[r, 0])) for r in range(3)]
            pz = p[2]
            xs, ys = p[0] / pz, p[1] / pz
            ix, iy = _coord(xs, W), _coord(ys, H)
            fx, fy = np.floor(ix), np.floor(iy)
            tx1, tx0 = (fx + f32(1)) - ix, ix - fx
            ty1, ty0 = (fy + f32(1)) - iy, iy - fy
            w = [tx1 * ty1, tx0 * ty1, tx1 * ty0, tx0 * ty0]
            X0, X1 = (fx >= 0) & (fx <= W - 1), (fx >= -1) & (fx <= W - 2)
            Y0, Y1 = (fy >= 0) & (fy <= H - 1), (fy >= -1) & (fy <= H - 2)
            xi = np.where(X0 | X1, fx, 0).astype(np.int64)
            yi = np.where(Y0 | Y1, fy, 0).astype(np.int64)
            ok = [X0 & Y0, X1 & Y0, X0 & Y1, X1 & Y1]
            off = [yi * W + xi, yi * W + xi + 1, (yi + 1) * W + xi, (yi + 1) * W + xi + 1]
            off = [np.where(o, a, 0) for o, a in zip(ok, off)]
            any_ = (X0 | X1) & (Y0 | Y1)
            vals = [[np.where(ok[k], planes[v, c][off[k]], f32(0)) for k in range(4)] for c in range(8)]
            for c in range(8):
                s = np.zeros(n, f32)
                for k in range(4):
                    s = np.where(ok[k], _fma(vals[c][k], w[k], s), s)
                feats[v, c] = s
            d = feats[v, 7] - pz
            feats[v, 7] = np.abs(d)
            sgn = np.where(d > 0, f32(1), np.where(d < 0, f32(-1), f32(0)))
            g_sd = g[v, 7] * sgn
            gix, giy = np.zeros(n, f32), np.zeros(n, f32)
            for c in range(8):
                go = g_sd if c == 7 else g[v, c]
                vv = vals[c]
                gix = _fma(go, (vv[1] - vv[0]) * ty1 + (vv[3] - vv[2]) * ty0, gix)
                giy = _fma(go, (vv[2] - vv[0]) * tx1 + (vv[3] - vv[1]) * tx0, giy)
                if c < 3:
                    continue
                for k in range(4):
                    m = ok[k] & (go != 0)
                    t = w[k] * go
                    if det:
                        s = t[m].astype(f64) * 2.0 ** kq
                        assert (np.abs(s) <= 2.0 ** (P.K_SUM_BITS - L)).all()
                        np.add.at(fixed[v, c - 3], off[k][m], np.rint(s).astype(np.int64))
                    else:
                        np.add.at(rend[v, c - 3], off[k][m], t[m])
            gxs = ((gix * f32(0.5 * W)) * f32(2)) / f32(W)
            gys = ((giy * f32(0.5 * H)) * f32(2)) / f32(H)
            dpx = np.where(any_, gxs / pz, f32(0))
            dpy = np.where(any_, gys / pz, f32(0))
            dpz = np.where(any_, -g_sd - (gxs * (xs / pz) + gys * (ys / pz)), -g_sd)
            dq = [_fma(dpz, Km[2, k], _fma(dpy, Km[1, k], dpx * Km[0, k])) for k in range(3)]
            dx = [_fma(dq[2], E[2, k], _fma(dq[1], E[1, k], dq[0] * E[0, k])) for k in range(3)]
            for k in range(3):
                gpt[:, k] = gpt[:, k] + dx[k]
    if det:
        rend = (fixed.astype(f32).astype(f64) * 2.0 ** -kq).astype(f32)
    return {"feats": feats, "g_points": gpt, "g_image": rend[:, :3].reshape(V, 3, H, W),
            "g_acc": rend[:, 3].reshape(V, H, W), "g_depth": rend[:, 4].reshape(V, H, W)}


# -------------------------------------------------------------------------------------------------------------- cases

def _camera(W, H, f=16.0):
    """An identity rotation at z = -2 and a pinhole with focal f and principal point 0: for a point (X, Y, 0),
    z = 2 and xs = f X / 2 exactly, and ix = xs exactly for 0 <= xs < 7.5 (every step of the chain is exact)."""
    w2c = torch.eye(4)[None].clone()
    w2c[0, 2, 3] = 2.0
    ixt = torch.tensor([[[f, 0.0, 0.0], [0.0, f, 0.0], [0.0, 0.0, 1.0]]])
    return w2c, ixt


def _images(V, H, W, seed, depth=None):
    g = torch.Generator().manual_seed(seed)
    img_ref = torch.rand((V, 3, H, W), generator=g)
    image = torch.rand((V, H, W, 3), generator=g)
    acc = torch.rand((V, H, W), generator=g)
    dep = (1.5 + torch.rand((V, H, W, 1), generator=g)) if depth is None else torch.full((V, H, W, 1), depth)
    return img_ref, {"image": image, "acc_map": acc, "depth": dep}


def _at(ix, iy, f=16.0):
    """Points (X, Y, 0) that _camera projects to (ix, iy), rounded to fp32."""
    return torch.stack([torch.as_tensor(ix, dtype=torch.float64) * 2 / f,
                        torch.as_tensor(iy, dtype=torch.float64) * 2 / f, torch.zeros(len(ix), dtype=torch.float64)],
                       1).float()


def border_case(H=24, W=20, seed=5):
    """Projections within one pixel outside each edge and corner (one or two taps valid), and just inside."""
    g = torch.Generator().manual_seed(seed)
    k = 400
    u = torch.rand(k, generator=g, dtype=torch.float64)
    w = torch.rand(k, generator=g, dtype=torch.float64)
    xs = [-u, W - 1 + u, -u, W - 1 + u, u * (W - 1), u * (W - 1), -0.999 * u, W - 1 + 0.999 * u]
    ys = [w * (H - 1), w * (H - 1), -w, H - 1 + w, -w, H - 1 + w, H - 1 + w, -w]
    w2c, ixt = _camera(W, H, f=float(W))
    pts = _at(torch.cat(xs), torch.cat(ys), f=float(W))
    img_ref, rend = _images(1, H, W, seed)
    return pts, img_ref, rend, w2c, ixt


def tiny_weight_case(H=16, W=16, seed=6):
    """ix, iy = j + 2^-20 and j + 1 - 2^-20 exactly, one point per cell: the pixels on the far side are reached only
    by weights of about 2^-20 (and 2^-40 at the far corner)."""
    t = 2.0 ** -20
    a = torch.tensor([0 + t, 2 + t, 4 + t, 7 - t], dtype=torch.float64)
    ix, iy = torch.meshgrid(a, a, indexing="ij")
    w2c, ixt = _camera(W, H)
    pts = _at(ix.reshape(-1), iy.reshape(-1))
    img_ref, rend = _images(1, H, W, seed)
    return pts, img_ref, rend, w2c, ixt


def tie_case(H=16, W=16, seed=7):
    """d = s_depth - z = 0 exactly: a constant depth plane 2, z = 2 exact, and weights 0.25 (ix, iy = j + 0.5)."""
    a = torch.arange(0, 7, dtype=torch.float64) + 0.5
    ix, iy = torch.meshgrid(a, a, indexing="ij")
    w2c, ixt = _camera(W, H)
    pts = _at(ix.reshape(-1), iy.reshape(-1))
    img_ref, rend = _images(1, H, W, seed, depth=2.0)
    return pts, img_ref, rend, w2c, ixt


def pile_up_case(n=100000, H=24, W=24, seed=8):
    """n points on three camera rays, the first two through neighbouring pixels, at depths 1 to 3 on both sides of the
    depth plane: single pixels of g_acc and g_depth sum about n terms."""
    g = torch.Generator().manual_seed(seed)
    w2c, ixt = _camera(W, H)
    rays = torch.tensor([[3.3, 4.6], [3.8, 4.4], [5.5, 2.25]], dtype=torch.float64)
    which = torch.arange(n) % 3
    s = 1.0 + 2.0 * torch.rand(n, generator=g, dtype=torch.float64)        # z_cam
    xy = rays[which] * 2 / 16.0 * s[:, None] / 2.0                          # X = xs z / f
    pts = torch.cat([xy, (s - 2.0)[:, None]], 1).float()
    img_ref, rend = _images(1, H, W, seed)
    return pts, img_ref, rend, w2c, ixt


def z_zero_case(seed=9):
    """test_point_in_camera_plane_samples_zero's scene: one point in the camera's plane among 300."""
    H, W, n = 40, 56, 300
    points, img_ref, rend, _, ixt = make_case(1, H, W, n, seed, behind=False)
    w2c = torch.eye(4)[None].clone()
    w2c[0, 2, 3] = 2.0
    points[150] = torch.tensor([0.3, -0.2, -2.0])
    return points, img_ref, rend, w2c, ixt[:1]


SPECIAL = {"border": border_case, "tiny_weights": tiny_weight_case, "ties": tie_case, "pile_up": pile_up_case,
           "z_zero": z_zero_case}


def _upstream(V, n, seed):
    return torch.randn((V, 8, n), generator=torch.Generator().manual_seed(seed))


def _case_specifics(name, case, st, res):
    """What each special case is built to show."""
    pts, img_ref, rend, w2c, ixt = case
    if name == "ties":
        assert (st["feats"].v[:, 7] == 0).all() and (st["feats"].e[:, 7] == 0).all()
        assert (np.asarray(res["feats"])[:, 7] == 0).all()
        assert (np.asarray(res["g_depth"]) == 0).all()          # sign(0) = 0: no channel-7 vjp at all
    if name == "tiny_weights":
        g = np.abs(st["g_image"].v)
        small = (g > 0) & (g < 1e-5)
        assert small.sum() >= 10, "no pixel reached only by tiny weights"
    if name == "pile_up":
        assert st["max_terms"] >= 60000, st["max_terms"]
    if name == "z_zero":
        assert not np.asarray(res["feats"])[:, :, 150].any() and not np.asarray(res["g_points"])[150].any()
        assert (st["feats"].e[:, :, 150] == 0).all() and (st["g_points"].e[150] == 0).all()
    if name == "border":
        f = st["feats"].v[0, 3]
        assert (f != 0).all(), "a border point outside the image's taps"


# ---------------------------------------------------------------------------------------------------------------- CPU

def _cpu_cases():
    return {"random": make_case(3, 48, 64, 2600, 11), "smooth": make_case(2, 40, 56, 1500, 12, coarse=8),
            **{k: f() for k, f in SPECIAL.items() if k != "pile_up"}}


@pytest.mark.parametrize("name", ["random", "smooth", "border", "tiny_weights", "ties"])
def test_statement_equals_torch_restatement_float64(name):
    """Values and gradients of point_feats_torch in float64 equal the statement's (its value at float64's decisions),
    to 1e-12 plus the double-rounding floor of the bound, wherever no decision is undecided.  (At z = 0 torch's result
    depends on how the non-finite coordinate converts; the kernels' designed rule is checked by the emulation.)"""
    case = _cpu_cases()[name]
    pts, img_ref, rend, w2c, ixt = case
    n, V = pts.shape[0], w2c.shape[0]
    up = _upstream(V, n, 1)
    st = statement(case, up)
    p = pts.double().requires_grad_(True)
    r = {k: v.double().requires_grad_(True) for k, v in rend.items()}
    out = point_feats_torch(p, img_ref.double(), r, w2c.double(), ixt.double())
    out.backward(up.double())
    wp = st["wide_pairs"]
    assert wp.mean() < 0.01
    _pin64(np.where(wp[:, None], 0.0, out.detach().numpy()), EB(np.where(wp[:, None], 0.0, st["feats"].v), st["feats"].e),
           "feats")
    keep = ~st["wide_points"]
    _pin64(p.grad.numpy()[keep], EB(st["g_points"].v[keep], st["g_points"].e[keep]), "g_points")
    gi, ga, gd = _planar({"image": r["image"].grad, "acc_map": r["acc_map"].grad, "depth": r["depth"].grad})
    for k, got, ch in (("g_image", gi, slice(0, 3)), ("g_acc", ga, 3), ("g_depth", gd, 4)):
        wpx = st["wide_pixels"][:, ch]
        ref = st[k]
        _pin64(np.where(wpx, 0.0, got), EB(np.where(wpx, 0.0, ref.v), ref.e), k)


@pytest.mark.parametrize("name", ["random", "smooth", "border", "tiny_weights", "ties"])
def test_fp32_torch_restatement_within_bound(name):
    case = _cpu_cases()[name]
    pts, img_ref, rend, w2c, ixt = case
    up = _upstream(w2c.shape[0], pts.shape[0], 2)
    st = statement(case, up)
    p = pts.clone().requires_grad_(True)
    r = {k: v.clone().requires_grad_(True) for k, v in rend.items()}
    out = point_feats_torch(p, img_ref, r, w2c, ixt)
    out.backward(up)
    gi, ga, gd = _planar({"image": r["image"].grad, "acc_map": r["acc_map"].grad, "depth": r["depth"].grad})
    res = {"feats": out.detach().numpy(), "g_points": p.grad.numpy(), "g_image": gi, "g_acc": ga, "g_depth": gd}
    check_all(res, st, False, f"fp32 torch {name}")


@pytest.mark.parametrize("name", ["random", "smooth", "border", "tiny_weights", "ties", "z_zero", "pile_up"])
def test_fp32_emulation_within_bound(name):
    """The kernels' sequence in fp32 NumPy, both summation modes, within the bound at every element."""
    case = SPECIAL[name]() if name == "pile_up" else _cpu_cases()[name]
    pts, img_ref, rend, w2c, ixt = case
    up = _upstream(w2c.shape[0], pts.shape[0], 3)
    st = statement(case, up)
    image, acc, depth = _planar(rend)
    for det in (False, True):
        res = emulate(pts.numpy(), w2c.numpy(), ixt.numpy(), img_ref.numpy(), image, acc, depth, up.numpy(), det)
        check_all(res, st, det, f"emulation {name} det={det}")
        _case_specifics(name, case, st, res)


def test_det_sum_restatement_matches_det_sum_cuh(host):
    """The host restatement of det_sum.cuh that the bound and the emulation use -- ceil_log2, scale_exp, the quantised
    term and the final conversion -- against det_sum.cuh itself, compiled for the host."""
    rng = np.random.default_rng(4)
    for n in (1, 2, 3, 4, 5, 255, 256, 257, 4096, 4097):
        x = np.zeros(n, f32)
        x[0] = f32(0.75)
        ok, _, k = _host_sum(host, x)
        assert ok and k == P.scale_exp(P.abs_bits_max(x), P.ceil_log2(n)), n
    for bits in [0, 1, 0x7FFFFF, 0x800000] + [int(b) for b in rng.integers(0, 0x7F800000, 200)]:
        for L in (0, 1, 5, 22, 24):
            assert host.h_scale_exp(bits, L) == P.scale_exp(bits, L), (bits, L)
    L = 22
    xs = (rng.standard_normal(500) * np.exp2(rng.integers(-30, 10, 500))).astype(f32)
    k = P.scale_exp(P.abs_bits_max(xs), L)
    for x in xs:
        q = ctypes.c_longlong()
        assert host.h_quantize(float(x), k, L, ctypes.byref(q)) == 1
        assert q.value == int(np.rint(f64(x) * 2.0 ** k)), x
    for S in [int(v) for v in rng.integers(-2 ** 62, 2 ** 62, 200)]:
        assert np.float32(host.h_to_float(S, k)) == f32(f64(f32(S)) * 2.0 ** -k), S


# ---------------------------------------------------------------------------------------------------------------- GPU

def _kernels(case, up, det, dev):
    from lara_b200.point_feats import sample_point_feats
    pts, img_ref, rend, w2c, ixt = case
    p = pts.to(dev).requires_grad_(True)
    r = {k: v.to(dev).requires_grad_(True) for k, v in rend.items()}
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        out = sample_point_feats(p, img_ref.to(dev), r, w2c.to(dev), ixt.to(dev))
        out.backward(up.to(dev))
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev)
    gi, ga, gd = _planar({"image": r["image"].grad, "acc_map": r["acc_map"].grad, "depth": r["depth"].grad})
    return {"feats": out.detach().cpu().numpy(), "g_points": p.grad.cpu().numpy(), "g_image": gi, "g_acc": ga,
            "g_depth": gd}


def _coverage(case):
    """At least one view each: a point outside, one partly outside, one behind a camera."""
    pts, img_ref, rend, w2c, ixt = case
    H, W = img_ref.shape[-2:]
    p = pts.double().numpy()
    cam = np.einsum("nk,vrk->vnr", p, w2c.double().numpy()[:, :3, :3]) + w2c.double().numpy()[:, None, :3, 3]
    z = cam[..., 2]
    assert (z < 0).any(), "no point behind a camera"
    pix = np.einsum("vnk,vrk->vnr", cam, ixt.double().numpy())
    with np.errstate(divide="ignore", invalid="ignore"):
        ix = pix[..., :2] / pix[..., 2:] - 0.5       # the sample coordinate, up to rounding
    inside = ((ix > 0) & (ix < np.array([W - 1, H - 1]))).all(-1)
    partly = ((ix > -1) & (ix < np.array([W, H]))).all(-1) & ~inside
    assert inside.any() and (~inside).any() and partly.any()


GPU_SHAPES = {"lara_4x262144_512": (4, 262144, 512, 512), "2x1000_80x96": (2, 1000, 80, 96), "1x1_32": (1, 1, 32, 32),
              "n0": (2, 0, 16, 24)}


@pytest.fixture(scope="module")
def gpu_statements():
    """The statement of each GPU case, computed once for both summation modes."""
    cache = {}

    def get(name):
        if name not in cache:
            if name in GPU_SHAPES:
                V, n, H, W = GPU_SHAPES[name]
                case = make_case(V, H, W, n, n + 1, coarse=8)
            else:
                case = SPECIAL[name]()
            up = _upstream(case[3].shape[0], case[0].shape[0], 17)
            cache[name] = (case, up, statement(case, up))
        return cache[name]
    return get


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("name", list(GPU_SHAPES) + list(SPECIAL))
def test_kernels_per_element(cuda_device, gpu_statements, name, det):
    case, up, st = gpu_statements(name)
    res = _kernels(case, up, det, cuda_device)
    assert res["feats"].shape == st["feats"].v.shape and res["g_points"].shape == (case[0].shape[0], 3)
    check_all(res, st, det, f"kernels {name} det={det}")
    _case_specifics(name, case, st, res)
    if name in GPU_SHAPES and GPU_SHAPES[name][1] > 1:
        _coverage(case)
