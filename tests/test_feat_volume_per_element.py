"""The coarse pass's feature-volume lifting (csrc/feat_volume.cu) element by element against float64.

``oracle.feat_volume64`` restates the kernels' operation sequence in float64 with a bound per element on what their fp32
evaluation may differ by (its docstring derives the rules; the taps are ``oracle.point_feats64``'s, shared with the
point sampler).  So a border token reached only by taps of small weight, a token whose dL/dx is small after the
LayerNorm vjp's cancellation and a small component of the ``mlp.1`` weight gradient are each held to their own bound,
not to a fraction of the tensor's largest element.  Where the bound leaves a voxel's ``floor(ix)`` or ``floor(iy)``
undecided, the element is held to the hull of both sides (the sample and every gradient are continuous there), and the
number of such voxel-views is printed.

CPU part: the statement equals the plain-torch restatement run in float64; the fp32 restatement and an fp32 NumPy
emulation of the kernels' operation sequence (strided LayerNorm sums, the gather's cell lists, per-CTA partials, the
view-embedding row slices) lie within the bound at every element.  GPU part: both layouts of the kernels, every output
and gradient, at LaRa's size and at ragged token tiles, grid sizes, channel counts, view-embedding widths, view and
group counts the kernels' tiling treats differently, a pile-up of every voxel in four cells, voxels on and a few ulps
from cell edges, and a voxel slice in a camera's plane.
"""
import math
import time

import numpy as np
import pytest
import torch

from oracle import feat_volume64 as F
from test_chain_per_element import _pin64, _tightness
from test_feat_volume import CPU, CPU_CASES, _kernel_run, make_case, torch_path
from test_point_feats_per_element import _check

f32, f64 = np.float32, np.float64
GRADS = ("g_img_feats", "g_norm_w", "g_norm_b", "g_mlp_w", "g_mlp_b", "g_view_embed")


# ---------------------------------------------------------------------------------------------------------- helpers

def _grid(R):
    from lara_b200.feat_volume import dense_grid
    return dense_grid(R)


def statement(case, dims, ups):
    """The statement of a case for the upstreams ups = [(n_group, tensor in that layout)], and its wall time."""
    B, V, C, R = dims
    img_feats, rays, w2c, ixt, params, ve, hw = case
    grads = [F.canonical(up, B, V, C, R, ng) for ng, up in ups]
    t0 = time.perf_counter()
    st = F.feat_volume64(img_feats, rays, w2c, ixt, hw, _grid(R), params, grads)
    st["seconds"] = time.perf_counter() - t0
    return st


def _ve(case):
    """view_embed [1,Vmax,E,1,1,1] of a case as [Vmax, E] (None without one)."""
    return None if case[5] is None else case[5].detach().reshape(case[5].shape[1], -1).numpy()


def _result(out, g_x, g_params, g_ve, ng, dims, V):
    """A run's outputs as arrays in the statement's form."""
    B, _, C, R = dims
    o, oe = F.canonical(out, B, V, C, R, ng)
    a = lambda t: t.detach().cpu().numpy().astype(f64)          # noqa: E731
    res = {"out": o, "out_ve": oe, "g_img_feats": a(g_x), "g_norm_w": a(g_params[0]), "g_norm_b": a(g_params[1]),
           "g_mlp_w": a(g_params[2]), "g_mlp_b": a(g_params[3])}
    if g_ve is not None:
        res["g_view_embed"] = a(g_ve).reshape(-1, oe.shape[-1])
    return res


def check_all(res, st, k, ve, ctx):
    """Every element of the run `res` (against upstream k of the statement) within its bound; the view-embedding columns
    are exact copies.  Prints the worst err/bound and the tightness; returns {output: worst err/bound}."""
    V = res["out"].shape[1]
    worst = {"out": _check(res["out"], st["out"], f"{ctx} out")}
    if res["out_ve"] is not None and res["out_ve"].shape[-1]:
        assert np.array_equal(res["out_ve"], np.broadcast_to(np.asarray(ve, f64)[None, :V, None], res["out_ve"].shape))
    g = st["grads"][k]
    for name in GRADS:
        if name not in g:
            continue
        got = res[name]
        if name == "g_view_embed":       # rows of views beyond V stay 0
            assert not got[V:].any()
            got = got[:V]
        worst[name] = _check(got, g[name], f"{ctx} {name}")
    print(f"\n  {ctx}: worst err/bound " + ", ".join(f"{n} {v:.3g}" for n, v in worst.items()) +
          f"; hulled voxel-views {int(st['hulled'].sum())}; most terms in one token {st['max_terms']}; "
          f"statement {st['seconds']:.1f} s")
    _tightness("out", st["out"])
    for name in GRADS:
        if name in g:
            _tightness(name, g[name])
    return worst


# ------------------------------------------------------------------------------------------- fp32 emulation (NumPy)

def _fma(a, b, c):
    """fmaf as one float64 operation rounded to fp32."""
    return (np.asarray(a, f64) * np.asarray(b, f64) + np.asarray(c, f64)).astype(f32)


def _rsh3(x, y, z):
    k = lambda v: f32(v)         # noqa: E731
    x2, y2, z2 = x * x, y * y, z * z
    c1, c2 = k(0.4886025119029199), k(1.0925484305920792)
    c9, c11 = k(0.5900435899266435), k(0.4570457994644658)
    return [np.full_like(x, k(0.28209479177387814)), -c1 * y, c1 * z, -c1 * x, c2 * (x * y), -c2 * (y * z),
            k(0.31539156525252005) * (f32(3) * z2 - f32(1)), -c2 * (x * z), k(0.5462742152960396) * (x2 - y2),
            (-c9 * y) * (f32(3) * x2 - y2), (k(2.890611442640554) * (x * y)) * z, (c11 * y) * (f32(1) - f32(5) * z2),
            (k(0.3731763325901154) * z) * (f32(5) * z2 - f32(3)), (c11 * x) * (f32(1) - f32(5) * z2),
            (k(1.445305721320277) * z) * (x2 - y2), (-c9 * x) * (x2 - f32(3) * y2)]


def _features(r):
    o, d = r[:, :3], r[:, 3:]
    inv = f32(1) / np.maximum(np.sqrt(_fma(d[:, 2], d[:, 2], _fma(d[:, 1], d[:, 1], d[:, 0] * d[:, 0]))), f32(1e-12))
    u = [d[:, k] * inv for k in range(3)]
    m = [o[:, 1] * u[2] - o[:, 2] * u[1], o[:, 2] * u[0] - o[:, 0] * u[2], o[:, 0] * u[1] - o[:, 1] * u[0]]
    f = np.stack(_rsh3(*u) + _rsh3(*m), 1)
    return f / (f32(1) + np.exp(-f))


def _butterfly(v):
    """warp_sum over the last axis (32 lanes): every lane ends with lane 0's value."""
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., lanes ^ o]
    return v[..., 0]


def _coord(xs, image_size, map_size):
    g = ((xs + f32(0.5)) / f32(image_size)) * f32(2) - f32(1)
    return ((g + f32(1)) * f32(map_size) - f32(1)) / f32(2)


def _taps(pts, E, K, h, w, H_img, W_img):
    x = [pts[:, k] for k in range(3)]
    with np.errstate(all="ignore"):
        q = [_fma(x[2], E[r, 2], _fma(x[1], E[r, 1], x[0] * E[r, 0])) + E[r, 3] for r in range(3)]
        p = [_fma(q[2], K[r, 2], _fma(q[1], K[r, 1], q[0] * K[r, 0])) for r in range(3)]
        ix, iy = _coord(p[0] / p[2], W_img, w), _coord(p[1] / p[2], H_img, h)
        fx, fy = np.floor(ix), np.floor(iy)
        tx1, tx0, ty1, ty0 = (fx + f32(1)) - ix, ix - fx, (fy + f32(1)) - iy, iy - fy
        X0, X1 = (fx >= 0) & (fx <= w - 1), (fx >= -1) & (fx <= w - 2)
        Y0, Y1 = (fy >= 0) & (fy <= h - 1), (fy >= -1) & (fy <= h - 2)
        xi, yi = np.where(X0 | X1, fx, 0).astype(np.int64), np.where(Y0 | Y1, fy, 0).astype(np.int64)
        cell = np.where((X0 | X1) & (Y0 | Y1), (yi + 1) * (w + 1) + xi + 1, -1)
    wts = np.stack([tx1 * ty1, tx0 * ty1, tx1 * ty0, tx0 * ty0], 1)
    ok = np.stack([X0 & Y0, X1 & Y0, X0 & Y1, X1 & Y1], 1)
    off = np.stack([yi * w + xi, yi * w + xi + 1, (yi + 1) * w + xi, (yi + 1) * w + xi + 1], 1)
    return wts, ok, np.where(ok, off, 0), cell


def emulate(case, dims, ng, up):
    """The kernels' operation sequence in fp32 (feat_volume.cu): token tiles of 64 with 8 tokens per warp, the cell
    lists ascending by voxel, per-CTA partials summed in fp64 in CTA order, view-embedding slices."""
    B, V, C, R = dims
    img_feats, rays, w2c, ixt, params, ve, (H_img, W_img) = case
    x = img_feats.numpy()
    BV, _, h, w = x.shape
    hw, R3, nj = h * w, R ** 3, C // 32
    ry, Es, Ks = rays.numpy().reshape(B, V, hw, 6), w2c.numpy(), ixt.numpy()
    gam, bet, W_, b_ = (p.numpy() for p in params)
    pts = _grid(R).numpy().reshape(-1, 3)
    G, GE = F.canonical(up, B, V, C, R, ng)
    G = G.astype(f32)
    ntiles = -(-hw // 64)
    out = np.zeros((B, V, R3, C), f32)
    gx = np.zeros((BV, C, hw), f32)
    parts = []
    for b in range(B):
        for v in range(V):
            bv = b * V + v
            xt = x[bv].reshape(C, hw)
            S = _features(ry[b, v])
            s = np.zeros((4, hw), f32)
            for q in range(C // 4):
                s = s + xt[4 * q:4 * q + 4]
            mean = (((s[0] + s[1]) + s[2]) + s[3]) / f32(C)
            s = np.zeros((4, hw), f32)
            for q in range(C // 4):
                d = xt[4 * q:4 * q + 4] - mean
                s = _fma(d, d, s)
            rstd = f32(1) / np.sqrt((((s[0] + s[1]) + s[2]) + s[3]) / f32(C) + f32(1e-6))
            sh = np.broadcast_to(b_[:C], (hw, C)).astype(f32)
            sc = np.broadcast_to(b_[C:], (hw, C)).astype(f32)
            for i in range(32):
                sh = _fma(W_[None, :C, i], S[:, i, None], sh)
                sc = _fma(W_[None, C:, i], S[:, i, None], sc)
            n = (xt.T - mean[:, None]) * rstd[:, None]
            ln = _fma(n, gam, bet)
            sc1 = f32(1) + sc
            y = _fma(ln, sc1, sh)
            wts, ok, off, cell = _taps(pts, Es[b, v], Ks[b, v], h, w, H_img, W_img)
            acc = np.zeros((R3, C), f32)
            for k in range(4):
                acc = np.where(ok[:, k, None], _fma(y[off[:, k]], wts[:, k, None], acc), acc)
            out[b, v] = acc
            # dL/dy: each token's four cells in order, each cell's voxels ascending
            order = np.argsort(np.where(cell >= 0, cell, np.iinfo(np.int64).max), kind="stable")
            ncell = (h + 1) * (w + 1)
            cnt = np.bincount(cell[cell >= 0], minlength=ncell)
            start = np.concatenate([[0], np.cumsum(cnt)])
            t = np.arange(hw)
            ty, tx = t // w, t % w
            W1 = w + 1
            dy = np.zeros((hw, C), f32)
            for k, cid in enumerate([(ty + 1) * W1 + tx + 1, (ty + 1) * W1 + tx, ty * W1 + tx + 1, ty * W1 + tx]):
                c_n, c_s = cnt[cid], start[cid]
                for r in range(int(c_n.max()) if hw else 0):
                    m = c_n > r
                    g = order[c_s[m] + r]
                    dy[m] = _fma(wts[g, k, None], G[b, v, g], dy[m])
            # token backward, tile by tile: warp wp holds the tokens wp + 8 j of the tile
            dsc, dln = dy * ln, dy * sc1
            dn = dln * gam
            for tile in range(ntiles):
                t0, nt = tile * 64, min(64, hw - tile * 64)
                aw = np.zeros((8, C, 32), f32)
                ac = np.zeros((8, C, 32), f32)
                rest = np.zeros((4, 8, C), f32)         # ab, abc, ag, abt
                for j in range(8):
                    for wp in range(8):
                        if wp + 8 * j >= nt:
                            continue
                        tk = t0 + wp + 8 * j
                        aw[wp] = _fma(dy[tk, :, None], S[tk][None], aw[wp])
                        ac[wp] = _fma(dsc[tk, :, None], S[tk][None], ac[wp])
                        rest[0, wp] = rest[0, wp] + dy[tk]
                        rest[1, wp] = rest[1, wp] + dsc[tk]
                        rest[2, wp] = _fma(dln[tk], n[tk], rest[2, wp])
                        rest[3, wp] = rest[3, wp] + dln[tk]
                tot = [aw[0], ac[0], rest[:, 0]]
                for wp in range(1, 8):
                    tot = [tot[0] + aw[wp], tot[1] + ac[wp], tot[2] + rest[:, wp]]
                parts.append(np.concatenate([tot[0].reshape(-1), tot[1].reshape(-1), tot[2].reshape(-1)]))
            s1 = np.zeros(hw, f32)
            s2 = np.zeros(hw, f32)
            dnn = dn * n
            for c0 in range(0, C, 32):
                s1 = s1 + _butterfly(dn[:, c0:c0 + 32])
                s2 = s2 + _butterfly(dnn[:, c0:c0 + 32])
            m1, m2 = s1 / f32(C), s2 / f32(C)
            gx[bv] = (rstd[:, None] * ((dn - m1[:, None]) - n * m2[:, None])).T
    tot = np.zeros(parts[0].size, f64)
    for p in parts:
        tot = tot + p.astype(f64)
    tot = tot.astype(f32)
    o = 2 * C * 32
    res = {"out": out, "out_ve": None if ng == 0 or not GE.shape[-1] else np.broadcast_to(_ve(case)[None, :V, None], GE.shape),
           "g_img_feats": gx.reshape(BV, C, h, w), "g_mlp_w": tot[:o].reshape(2 * C, 32),
           "g_mlp_b": tot[o:o + 2 * C], "g_norm_w": tot[o + 2 * C:o + 3 * C], "g_norm_b": tot[o + 3 * C:o + 4 * C]}
    if ng > 0 and GE.shape[-1]:
        E = GE.shape[-1]
        bs3 = (R // ng) ** 3
        rows = F.cond_rows(B, V, R, ng)
        flat = np.zeros((B * ng ** 3 * V * bs3, E), f32)
        flat[rows.reshape(-1)] = GE.reshape(-1, E)
        n = B * R3
        gve = np.zeros((V, E), f32)
        for v in range(V):
            total = np.zeros(E, f64)
            for z in range(64):
                lo, hi = n * z // 64, n * (z + 1) // 64
                red = []
                for grp in range(8):
                    s = np.zeros(E, f32)
                    for j in range(lo + grp, hi, 8):
                        s = s + flat[(j // bs3 * V + v) * bs3 + j % bs3]
                    red.append(s)
                t_ = np.zeros(E, f32)
                for r_ in red:
                    t_ = t_ + r_
                total = total + t_.astype(f64)
            gve[v] = total.astype(f32)
        res["g_view_embed"] = gve
    return res


# ---------------------------------------------------------------------------------------------------------------- CPU

# B, V, C, (h, w), (H_img, W_img), R, E, n_group, straddle: h w = 99 tokens (a last tile of 35), R = 5
CPU_RAGGED = (1, 2, 64, (9, 11), (144, 176), 5, 3, 1, False)


def _cpu_case(name):
    if name == "ragged":
        B, V, C, (h, w), hw, R, E, ng, straddle = CPU_RAGGED
        seed = 58
    else:
        ng, E, straddle = CPU_CASES[name]
        B, V, C, h, w, R, hw = CPU["B"], CPU["V"], CPU["C"], CPU["h"], CPU["w"], CPU["R"], (CPU["H"], CPU["W"])
        seed = 31 + len(name)
    case = make_case(B, V, C, h, w, hw[0], hw[1], R, E, seed, straddle) + (hw,)
    shape = (B, V, C, R, R, R) if ng == 0 else (B * ng ** 3, V * (R // ng) ** 3, C + E)
    up = torch.randn(shape, generator=torch.Generator().manual_seed(7))
    return case, (B, V, C, R), ng, up


CPU_NAMES = sorted(CPU_CASES) + ["ragged"]


def _torch_run(case, dims, ng, up, dtype):
    img_feats, rays, w2c, ixt, params, ve, hw = case
    x = img_feats.to(dtype).clone().requires_grad_(True)
    ps = [p.to(dtype).clone().requires_grad_(True) for p in params]
    v = ve.to(dtype).clone().requires_grad_(True) if (ve is not None and ng > 0) else None
    out = torch_path(x, rays.to(dtype), w2c.to(dtype), ixt.to(dtype), hw, _grid(dims[3]).to(dtype), ps, v, ng)
    out.backward(up.to(dtype))
    return _result(out, x.grad, [p.grad for p in ps], None if v is None else v.grad.reshape(v.shape[1], -1), ng, dims,
                   dims[1])


@pytest.mark.parametrize("name", CPU_NAMES)
def test_statement_equals_torch_restatement_float64(name):
    """The statement's value is feat_volume_torch's in float64, to 1e-12 plus the double-rounding floor of the bound."""
    case, dims, ng, up = _cpu_case(name)
    st = statement(case, dims, [(ng, up)])
    assert not st["hulled"].any()
    res = _torch_run(case, dims, ng, up, torch.float64)
    _pin64(res["out"], st["out"], "out")
    for k, ref in st["grads"][0].items():
        got = res[k][:dims[1]] if k == "g_view_embed" else res[k]
        _pin64(got, ref, k)


@pytest.mark.parametrize("name", CPU_NAMES)
def test_fp32_torch_restatement_within_bound(name):
    case, dims, ng, up = _cpu_case(name)
    st = statement(case, dims, [(ng, up)])
    res = _torch_run(case, dims, ng, up, torch.float32)
    check_all(res, st, 0, _ve(case), f"fp32 torch {name}")


@pytest.mark.parametrize("name", CPU_NAMES)
def test_fp32_emulation_within_bound(name):
    case, dims, ng, up = _cpu_case(name)
    st = statement(case, dims, [(ng, up)])
    res = emulate(case, dims, ng, up)
    check_all(res, st, 0, _ve(case), f"emulation {name}")


# ---------------------------------------------------------------------------------------------------------------- GPU

def _edge_camera(sx, sy, ex, ey):
    """An identity rotation at z = 2.03125 and focal 512: the voxel slice 7 of R = 16 has z = 2 exactly, and its voxel
    (i, j) projects to ix = i + sx + 16 ex, iy = j + sy + 16 ey on a 32 x 32 map of a 512 x 512 image, every step of
    the chain exact for ex, ey in {0, 2^-23, 2^-6} -- on cell edges (cells -1 and w - 1 among them), one step of the
    chain's resolution off them (ix = -1 + 2^-19: the voxel's only taps weigh 2^-19 ty), or a quarter cell off."""
    w2c = torch.eye(4)
    w2c[:3, 3] = torch.tensor([ex, ey, 2.03125])
    ixt = torch.tensor([[512.0, 0.0, 16 * sx + 127.5], [0.0, 512.0, 16 * sy + 127.5], [0.0, 0.0, 1.0]])
    return w2c, ixt


def _pile_up(case, W_img, H_img):
    """Every camera with focal 4 image pixels and its principal point inside one token cell: each view's voxels fall in
    at most 4 cells."""
    ixt = case[3].clone()
    ixt[..., 0, 0] = ixt[..., 1, 1] = 4.0
    ixt[..., 0, 2], ixt[..., 1, 2] = W_img / 2 + 5.3, H_img / 2 - 3.1
    return case[:3] + (ixt,) + case[4:]


def _border_ties(case):
    """Views 0 and 1 of each scene as make_case's straddling cameras; views 2 and 3 edge cameras: exactly on the edges,
    2^-19 inside cell -1 in x with taps of weight 2^-21 (scene 0), and a few ulps off the edges with rounding in the
    chain, so that the bound leaves floor(ix) undecided (scene 1)."""
    w2c, ixt = case[2].clone(), case[3].clone()
    for b in range(w2c.shape[0]):
        w2c[b, 2], ixt[b, 2] = _edge_camera(16, -15, 0.0, 0.0)
        w2c[b, 3], ixt[b, 3] = _edge_camera(-15, 16, 2.0 ** -23, 2.0 ** -6) if b == 0 else \
            _edge_camera(-15, 16, 3 * 2.0 ** -24, 3 * 2.0 ** -24)
    return case[:2] + (w2c, ixt) + case[4:]


# B, V, C, (h, w), (H_img, W_img), R, E, n_group, straddle
GPU_CASES = {
    "lara": (3, 4, 768, (32, 32), (512, 512), 16, 32, 16, False),
    "ragged": (2, 3, 64, (23, 37), (368, 592), 15, 33, 5, False),
    "tiny": (1, 8, 32, (5, 7), (80, 112), 5, 1, 1, False),
    "wide": (1, 2, 1024, (16, 16), (256, 256), 8, 128, 2, False),
    "v1_g4": (2, 1, 768, (32, 32), (512, 512), 16, 32, 4, False),
    "r64": (1, 2, 32, (32, 32), (512, 512), 64, 0, 4, False),
    "pile_up": (1, 2, 96, (20, 20), (320, 320), 15, 8, 3, False),
    "border_ties": (2, 4, 384, (32, 32), (512, 512), 16, 32, 8, True),
}


def _gpu_case(name):
    B, V, C, (h, w), hw, R, E, ng, straddle = GPU_CASES[name]
    case = make_case(B, V, C, h, w, hw[0], hw[1], R, E, 200 + len(name), straddle)
    if case[5] is not None and case[5].shape[1] < V:         # a view_embed row per view
        ve = torch.randn((1, V, E, 1, 1, 1), generator=torch.Generator().manual_seed(6)) / E ** 0.5
        case = case[:5] + (ve,)
    if name == "pile_up":
        case = _pile_up(case, hw[1], hw[0])
    if name == "border_ties":
        case = _border_ties(case)
    g = torch.Generator().manual_seed(5)
    ups = [(layout, torch.randn((B, V, C, R, R, R) if layout == 0 else (B * layout ** 3, V * (R // layout) ** 3, C + E),
                                generator=g)) for layout in (0, ng)]
    return case + (hw,), (B, V, C, R), ups


def _plane_case():
    """One camera (w2c = [I | -z_k]) whose plane holds the voxel slice k = 3 of R = 16."""
    C, h, w, H, W, R, k = 384, 32, 32, 512, 512, 16, 3
    case = list(make_case(1, 1, C, h, w, H, W, R, 0, 77))
    zk = float(_grid(R)[0, 0, k, 2])
    w2c = torch.eye(4)
    w2c[2, 3] = -zk
    case[2] = w2c.view(1, 1, 4, 4)
    f = 0.5 * W / math.tan(0.4)
    case[3] = torch.tensor([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]]).view(1, 1, 3, 3)
    up = torch.randn((1, 1, C, R, R, R), generator=torch.Generator().manual_seed(3))
    return tuple(case) + ((H, W),), (1, 1, C, R), [(0, up)], k


@pytest.fixture(scope="module")
def gpu_statements():
    """The statement of each GPU case, computed once for both layouts."""
    cache = {}

    def get(name):
        if name not in cache:
            case, dims, ups = _gpu_case(name)[:3] if name != "plane" else _plane_case()[:3]
            cache[name] = (case, dims, ups, statement(case, dims, ups))
        return cache[name]
    return get


def _module(case, C, R, dev):
    from lara_b200.feat_volume import FeatVolume
    params, ve = case[4], case[5]
    E = 0 if ve is None else ve.shape[2]
    fv = FeatVolume(C, E, R, n_views=4 if ve is None else ve.shape[1]).to(dev)
    with torch.no_grad():
        for p, v in zip((fv.dir_norm.norm.weight, fv.dir_norm.norm.bias, fv.dir_norm.mlp[1].weight,
                         fv.dir_norm.mlp[1].bias), params):
            p.copy_(v)
        if E > 0:
            fv.view_embed.copy_(ve)
    return fv


def _kernels(case, dims, ng, up, dev):
    B, V, C, R = dims
    fv = _module(case, C, R, dev)
    runs = _kernel_run(fv, case[:6], case[6], ng, up.to(dev), dev)
    g_ve = runs[6] if len(runs) > 6 else None
    return _result(runs[0], runs[1], runs[2:6], None if g_ve is None else g_ve.reshape(g_ve.shape[1], -1), ng, dims, V), \
        runs[0]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GPU_CASES))
def test_kernels_per_element(cuda_device, gpu_statements, name):
    from oracle.feat_volume_torch import cond_tokens_torch
    case, dims, ups, st = gpu_statements(name)
    ve = _ve(case)
    outs = {}
    for k, (ng, up) in enumerate(ups):
        res, outs[ng] = _kernels(case, dims, ng, up, cuda_device)
        check_all(res, st, k, ve, f"kernels {name} layout {ng}")
    # the two layouts hold the same bits
    ng = ups[1][0]
    ve_t = None if case[5] is None else case[5].to(cuda_device)
    assert torch.equal(cond_tokens_torch(outs[0], ve_t, ng), outs[ng])
    if name == "pile_up":
        assert st["max_terms"] >= 3000, st["max_terms"]
    if name == "border_ties":
        assert st["hulled"].any(), "no voxel a few ulps from a cell edge"


@pytest.mark.gpu
def test_kernels_voxel_in_a_camera_plane(cuda_device, gpu_statements):
    """The voxel slice in the camera's plane samples exactly 0 and passes no gradient (the statement gives it no tap and
    a zero bound); every other element is held to its bound."""
    case, dims, ups, st = gpu_statements("plane")
    k = _plane_case()[3]
    res, out = _kernels(case, dims, 0, ups[0][1], cuda_device)
    assert not bool(out[..., k].any())
    sl = np.zeros((16, 16, 16), bool)
    sl[..., k] = True
    sl = sl.reshape(-1)
    assert (st["out"].v[:, :, sl] == 0).all() and (st["out"].e[:, :, sl] == 0).all()
    check_all(res, st, 0, None, "kernels camera plane")
