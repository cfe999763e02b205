"""Float64 statement, with a bound per element, of the fine pass's point-feature sampler (lara_b200/csrc/point_feats.cu),
forward and backward.

TEST INFRASTRUCTURE ONLY -- importable from tests/; never from lara_b200/.

Every value is an ``oracle.EB``: the float64 value of the kernels' formula and a bound on what any fp32 evaluation of
it may differ by.  Each correctly rounded fp32 operation adds half an ulp of its result, ``U (|v| + e)``, and nothing
where its operands are exact and the result is an fp32 value (chain64's ``_exact`` rule, and 0 + x).  The short sums --
the projection's and its vjp's 3- and 4-term dot products, the vjp's three z terms and the sum over the views -- carry
the order-free bound ``(m - 1) U sum |term|``, so a matmul that adds in another order or with FMA stays inside it.

The sample coordinate ``ix`` is not used with an independent bound on each weight: its error moves the four weights
together.  Given the cell ``floor(ix)``, everything the kernels form from the weights -- the 8-channel sample, each tap's
``w``, and ``gix`` / ``giy`` -- is bilinear in the computed (ix, iy), so over the box ``ix +- e_ix``, ``iy +- e_iy``
its range is spanned by the box's corners.  Each corner is evaluated with its own rounding bound; the element's bound
is the corners' spread around the value plus the largest rounding bound.  ``tx0 = ix - fx`` and ``tx1 = fx + 1 - ix``
are exact by Sterbenz except in the cells -1 and 0 (where ``1 - ix`` or ``ix + 1`` round).

Decisions.  ``floor(ix)`` (which also decides each border tap's in/out test) is undecided where the box straddles an
integer, and ``sign(s_depth - z)`` where the range of ``d`` reaches 0.  Such a pair is not excluded: every side is
evaluated and the element is held to the hull of all of them, its midpoint with the half-range added to the bound.
Features and rendering gradients are continuous across the cell boundary, so their hull stays tight; the point gradient
jumps there, and its hull is wide.  These elements are counted (``widened``).  A box that spans more than two cells
inside the image, or a ``|z|`` whose bound reaches 0, gets an infinite bound (``inf_pairs``); z = 0 exactly (no error)
is decided: the coordinate is not finite, no tap is used, the point samples 0.

Rendering gradients: each pixel's terms ``w go`` are scattered with ``np.bincount``; the bound is the sum of the terms'
bounds plus, for ``red.global.add.f32`` in any order, ``gamma(m - 1) sum |term|`` over the m terms the pixel receives,
or in deterministic mode det_sum.cuh's own error ``m 2^-(k+1)`` and the final fp32 rounding, with k from the actual
``max |g_feats|`` and ``L = ceil_log2(4 V n)`` as the kernels compute them.
"""
from __future__ import annotations

from itertools import combinations

import numpy as np

from .oracle import EB

U = 2.0 ** -24                  # half an ulp, relative: one correctly rounded fp32 operation
SUB_ULP = 2.0 ** -149
K_SUM_BITS = 62                 # det_sum.cuh's kSumBits
_DX = (0, 1, 0, 1)              # tap k of a cell: nw, ne, sw, se
_DY = (0, 0, 1, 1)


def _rep(v):
    with np.errstate(over="ignore", invalid="ignore"):
        return v.astype(np.float32).astype(np.float64) == v


def _zero(a: EB):
    return (a.v == 0) & (a.e == 0)


def _round(v, e, exact):
    """The result of one fp32 operation: the operands' propagated bound e, plus half an ulp unless it is exact."""
    with np.errstate(invalid="ignore"):
        return EB(v, np.where(exact, e, e + U * (np.abs(v) + e)))


def add(a, b) -> EB:
    a, b = EB.w(a), EB.w(b)
    v, e = a.v + b.v, a.e + b.e
    return _round(v, e, ((a.e == 0) & (b.e == 0) & _rep(v)) | _zero(a) | _zero(b))


def mul(a, b) -> EB:
    a, b = EB.w(a), EB.w(b)
    with np.errstate(invalid="ignore"):
        v = a.v * b.v
        e = np.abs(a.v) * b.e + np.abs(b.v) * a.e + a.e * b.e
    return _round(v, e, (a.e == 0) & (b.e == 0) & _rep(v))


def div(a, b) -> EB:
    a, b = EB.w(a), EB.w(b)
    with np.errstate(divide="ignore", invalid="ignore"):
        v = a.v / b.v
        den = np.abs(b.v) - b.e
        e = np.where(den > 0, (a.e + np.abs(v) * b.e) / np.where(den > 0, den, 1.0), np.inf)
    return _round(v, e, (a.e == 0) & (b.e == 0) & (b.v != 0) & _rep(v))


def scale(a: EB, s: float) -> EB:
    """Multiplication by a power of two: exact."""
    return EB(a.v * s, a.e * abs(s))


def sum_any_order(terms) -> EB:
    """fp32 sum of the terms in any order and association (FMA included when the terms are products): the terms'
    bounds plus (m - 1) U (sum |term| + bounds) for the m terms that are not an exact 0; exact where every term and
    every partial sum in any order is an exact fp32 value."""
    terms = [EB.w(t) for t in terms]
    v = sum(t.v for t in terms)
    e = sum(t.e for t in terms)
    mag = sum(np.abs(t.v) + t.e for t in terms)
    m = sum((~_zero(t)).astype(np.float64) for t in terms)
    exact = np.ones(np.broadcast(*[t.v for t in terms]).shape, bool)
    for t in terms:
        exact = exact & (t.e == 0)
    for r in range(2, len(terms) + 1):
        for c in combinations(terms, r):
            exact = exact & _rep(sum(t.v for t in c))
    g = np.maximum(m - 1, 0) * U
    return EB(v, np.where(exact, 0.0, e + g / (1 - g) * mag))


def dot(pairs) -> EB:
    return sum_any_order([mul(a, b) for a, b in pairs])


def source_coord(xs: EB, image_size: int, map_size: int = None) -> EB:
    """network.py:401 (the normalisation by the image size), then grid_sample's unnormalisation onto a map of map_size
    pixels (align_corners=False), one rounding per torch operation: sample_taps.cuh's pf_source_coord.  The point
    sampler samples maps of the image's size."""
    map_size = image_size if map_size is None else map_size
    b = div(add(xs, 0.5), float(image_size))
    g = add(scale(b, 2.0), -1.0)
    return scale(add(mul(add(g, 1.0), float(map_size)), -1.0), 0.5)


def _f64(a):
    if hasattr(a, "detach"):
        a = a.detach().cpu().numpy()
    return np.asarray(a, dtype=np.float32).astype(np.float64)


# --------------------------------------------------------------------------------------------------------- one view

class _View:
    """One source view: the projection of every point with its bound, and the decisions of floor(ix), floor(iy) on a
    W x H map (of an image of W_img x H_img pixels, by default the map's size)."""

    def __init__(self, pts, E, Km, W, H, W_img=None, H_img=None):
        x = [EB(pts[:, k]) for k in range(3)]
        q = [sum_any_order([mul(x[0], E[r, 0]), mul(x[1], E[r, 1]), mul(x[2], E[r, 2]), EB.w(E[r, 3])])
             for r in range(3)]
        p = [dot([(q[0], Km[r, 0]), (q[1], Km[r, 1]), (q[2], Km[r, 2])]) for r in range(3)]
        self.pz = p[2]
        self.xs, self.ys = div(p[0], p[2]), div(p[1], p[2])
        self.zero = _zero(p[2])                       # z = 0 exactly: coordinates not finite, decided
        self.ix = source_coord(self.xs, W if W_img is None else W_img, W)
        self.iy = source_coord(self.ys, H if H_img is None else H_img, H)
        self.ax = self._axis(self.ix, W)
        self.ay = self._axis(self.iy, H)
        with np.errstate(invalid="ignore"):
            bad_pz = ~(np.abs(self.pz.v) > self.pz.e) & ~self.zero
        out = self.ax["out"] | self.ay["out"]
        self.inf = bad_pz | (~out & (self.ax["wide"] | self.ay["wide"] | self.ax["bad"] | self.ay["bad"]))
        # a pair with no tap in either axis, or an infinite bound, is evaluated with no taps
        for a in (self.ax, self.ay):
            for k in ("cA", "cB", "c0"):
                a[k] = np.where(out | self.inf, -8.0, a[k])
            a["und"] = a["und"] & ~out & ~self.inf

    def _axis(self, c: EB, size):
        fin = np.isfinite(c.v) & np.isfinite(c.e) & ~self.zero
        v, e = np.where(fin, c.v, 0.0), np.where(fin, c.e, 0.0)
        lo, hi = np.floor(v - e), np.floor(v + e)
        out = ~fin | (hi < -1) | (lo > size - 1)
        return dict(v=v, ex=fin & (c.e == 0), cA=lo, cB=hi, c0=np.floor(v), lo=v - e, hi=v + e, out=out & (self.zero | fin),
                    bad=~fin & ~self.zero, wide=(hi - lo >= 2), und=(hi - lo == 1))


def _positions(a, idx, undecided):
    """[(cell, position)] spanning the box of axis `a` over the pairs idx: its two ends in the cell, or with an undecided
    floor the ends in each of the two cells (an axis that is decided repeats its cell)."""
    cA, cB, lo, hi = a["cA"][idx], a["cB"][idx], a["lo"][idx], a["hi"][idx]
    if not undecided:
        return [(cA, np.clip(lo, cA, cA + 1)), (cA, np.clip(hi, cA, cA + 1))]
    u = a["und"][idx]
    cB = np.where(u, cB, cA)
    return [(cA, np.clip(lo, cA, cA + 1)), (cA, np.clip(np.where(u, cA + 1, hi), cA, cA + 1)),
            (cB, np.clip(np.where(u, cB, lo), cB, cB + 1)), (cB, np.clip(hi, cB, cB + 1))]


def _weights(cx, px, ex, cy, py, ey):
    """tx0, tx1, ty0, ty1 of the kernel at the exact computed coordinates (px, py) of the cells (cx, cy); ex / ey:
    the coordinate is an exact fp32 value, so a difference that is an fp32 value is exact in the cells -1 and 0 too."""
    def axis(c, p, exact):
        t0, t1 = p - c, c + 1.0 - p
        r0 = np.where((c < 0) & ~(exact & _rep(t0)), U * np.abs(t0), 0.0)
        r1 = np.where(((c == 0) | (c == -1)) & ~(exact & _rep(t1)), U * np.abs(t1), 0.0)
        return EB(t0, r0), EB(t1, r1)
    tx0, tx1 = axis(cx, px, ex)
    ty0, ty1 = axis(cy, py, ey)
    return tx0, tx1, ty0, ty1


class _Hull:
    """Running range of the values over the evaluated sides and the largest rounding bound."""

    def __init__(self):
        self.lo = self.hi = self.r = None

    def add(self, x: EB):
        if self.lo is None:
            self.lo, self.hi, self.r = x.v.copy(), x.v.copy(), x.e.copy()
        else:
            self.lo, self.hi, self.r = np.minimum(self.lo, x.v), np.maximum(self.hi, x.v), np.maximum(self.r, x.e)


def _valid(cx, cy, W, H):
    """The four taps' in-image tests of the cells (cx, cy)."""
    return [(cx + _DX[k] >= 0) & (cx + _DX[k] <= W - 1) & (cy + _DY[k] >= 0) & (cy + _DY[k] <= H - 1) for k in range(4)]


def _stencil_hull(vw, idx, xs, ys, W, H):
    """Hulls, over every (x side, y side) combination of the pairs idx, of the weight each slot of the 3x3 stencil
    around the lower candidate cell (cA, cA) receives (0 where a combination's taps miss the slot), and the slots some
    combination taps."""
    m = idx.size
    baseX, baseY = vw.ax["cA"][idx], vw.ay["cA"][idx]
    exx, exy = vw.ax["ex"][idx], vw.ay["ex"][idx]
    wst = [_Hull() for _ in range(9)]
    touched = np.zeros((9, m), bool)
    for cx, px in xs:
        for cy, py in ys:
            tx0, tx1, ty0, ty1 = _weights(cx, px, exx, cy, py, exy)
            w = [mul(tx1, ty1), mul(tx0, ty1), mul(tx1, ty0), mul(tx0, ty0)]
            valid = _valid(cx, cy, W, H)
            sv, se = np.zeros((9, m)), np.zeros((9, m))
            for k in range(4):
                slot = ((cy - baseY + _DY[k]) * 3 + (cx - baseX + _DX[k])).astype(np.int64)
                for s_ in range(9):
                    here = valid[k] & (slot == s_)
                    touched[s_] |= here
                    sv[s_] = np.where(here, w[k].v, sv[s_])
                    se[s_] = np.where(here, w[k].e, se[s_])
            for s_ in range(9):
                wst[s_].add(EB(sv[s_], se[s_]))
    return wst, touched


def stencil(vw, W, H, und):
    """The tap weight each slot s of the 3x3 stencil around every pair's lower candidate cell receives, for both
    statements: ``touched`` [9,n] (some side of the pair's box taps the slot), the slot's pixel ``X``, ``Y`` [9,n]
    (cA + s % 3, cA + s // 3), and the weight as a value ``v`` with its spread ``d`` over the box and a rounding bound
    ``r`` [9,n]: any weight an fp32 evaluation gives lies within v +- (d + r).  A decided pair (und False) takes the
    value at the float64 coordinates and the corners' largest distance from it; an undecided one the hull of every
    side, its midpoint and half-range."""
    n = vw.ax["v"].size
    allidx = np.arange(n)
    c0x, c0y = vw.ax["c0"], vw.ay["c0"]
    cen, _ = _stencil_hull(vw, allidx, [(c0x, np.clip(vw.ax["v"], c0x, c0x + 1))],
                           [(c0y, np.clip(vw.ay["v"], c0y, c0y + 1))], W, H)
    out = {k: np.zeros((9, n)) for k in ("v", "d", "r")}
    out["touched"] = np.zeros((9, n), bool)
    for sub, u in ((allidx[~und], False), (allidx[und], True)):
        if sub.size == 0:
            continue
        hull, touched = _stencil_hull(vw, sub, _positions(vw.ax, sub, u), _positions(vw.ay, sub, u), W, H)
        for s_ in range(9):
            h = hull[s_]
            out["touched"][s_, sub] = touched[s_]
            if u:
                out["v"][s_, sub], out["d"][s_, sub], out["r"][s_, sub] = 0.5 * (h.lo + h.hi), 0.5 * (h.hi - h.lo), h.r
            else:
                c = cen[s_].lo[sub]
                out["v"][s_, sub], out["d"][s_, sub] = c, np.maximum(h.hi - c, c - h.lo)
                out["r"][s_, sub] = np.maximum(h.r, cen[s_].r[sub])
    s = np.arange(9)[:, None]
    out["X"], out["Y"] = vw.ax["cA"][None] + s % 3, vw.ay["cA"][None] + s // 3
    return out


def _eval(planes, vw, idx, xs, ys, signs, g, W, H, want_grad, Km, E, only_d=False):
    """Evaluate the pairs idx at every (x side, y side, sign) combination.  planes [8,H*W] float64 of the view,
    g [8,n] the view's upstream (or None).  Returns hulls of the features [8], d = s_depth - z, and the point gradient
    [3]."""
    m = idx.size
    exx, exy = vw.ax["ex"][idx], vw.ay["ex"][idx]
    pz = EB(vw.pz.v[idx], vw.pz.e[idx])
    xsE, ysE = EB(vw.xs.v[idx], vw.xs.e[idx]), EB(vw.ys.v[idx], vw.ys.e[idx])
    feats = [_Hull() for _ in range(8)]
    dh = _Hull()
    grad = [_Hull() for _ in range(3)]
    Wf, Hf = float(W), float(H)
    for cx, px in xs:
        for cy, py in ys:
            tx0, tx1, ty0, ty1 = _weights(cx, px, exx, cy, py, exy)
            w = [mul(tx1, ty1), mul(tx0, ty1), mul(tx1, ty0), mul(tx0, ty0)]
            valid = _valid(cx, cy, W, H)
            vals = []
            for k in range(4):
                off = np.where(valid[k], (cy + _DY[k]) * W + cx + _DX[k], 0).astype(np.int64)
                vals.append(np.where(valid[k][None], planes[:, off], 0.0))         # [8, m]
            any_ = (((cx >= 0) & (cx <= W - 1)) | ((cx >= -1) & (cx <= W - 2))) & \
                (((cy >= 0) & (cy <= H - 1)) | ((cy >= -1) & (cy <= H - 2)))
            samp = []
            for c in ([7] if only_d else range(8)):
                s = EB(np.zeros(m))
                for k in range(4):
                    s = EB.where(valid[k], add(s, mul(EB(vals[k][c]), w[k])), s)
                samp.append(s)
            d = add(samp[-1], -pz)
            dh.add(EB(d.v, d.e))
            if only_d:
                continue
            for c in range(7):
                feats[c].add(samp[c])
            if not want_grad:
                continue
            for sg in signs:
                gix, giy = EB(np.zeros(m)), EB(np.zeros(m))
                for c in range(8):
                    go = EB(g[c, idx] * sg) if c == 7 else EB(g[c, idx])
                    v0, v1, v2, v3 = (EB(vals[k][c]) for k in range(4))
                    gix = add(gix, mul(go, add(mul(add(v1, -v0), ty1), mul(add(v3, -v2), ty0))))
                    giy = add(giy, mul(go, add(mul(add(v2, -v0), tx1), mul(add(v3, -v1), tx0))))
                g_sd = EB(g[7, idx] * sg)
                gxs = div(scale(mul(gix, 0.5 * Wf), 2.0), Wf)
                gys = div(scale(mul(giy, 0.5 * Hf), 2.0), Hf)
                dpx, dpy = div(gxs, pz), div(gys, pz)
                dpz = sum_any_order([-g_sd, -mul(gxs, div(xsE, pz)), -mul(gys, div(ysE, pz))])
                zero = EB(np.zeros(m))
                dpx, dpy, dpz = EB.where(any_, dpx, zero), EB.where(any_, dpy, zero), EB.where(any_, dpz, -g_sd)
                dq = [dot([(dpx, Km[0, k]), (dpy, Km[1, k]), (dpz, Km[2, k])]) for k in range(3)]
                dx = [dot([(dq[0], E[0, k]), (dq[1], E[1, k]), (dq[2], E[2, k])]) for k in range(3)]
                for k in range(3):
                    grad[k].add(dx[k])
    if not only_d:      # |d| over the range of d: 0 where the range holds 0 (|d| is least inside the box there)
        h = feats[7]
        h.hi, h.r = np.maximum(np.abs(dh.lo), np.abs(dh.hi)), dh.r
        h.lo = np.where((dh.lo <= 0) & (dh.hi >= 0), 0.0, np.minimum(np.abs(dh.lo), np.abs(dh.hi)))
    return dict(feats=feats, d=dh, grad=grad)


def _sign_set(d: _Hull):
    lo, hi = d.lo - d.r, d.hi + d.r
    smin = np.where(lo < 0, -1.0, np.where(lo == 0, 0.0, 1.0))
    smax = np.where(hi > 0, 1.0, np.where(hi == 0, 0.0, -1.0))
    return smin, smax


def point_feats64(points, w2cs, ixts, img_ref, image, acc, depth, g_feats=None):
    """The sampler's outputs as EB: ``feats`` [V,8,n]; with ``g_feats`` [V,8,n] also ``g_points`` [n,3], and the
    rendering gradients ``g_image`` [V,3,H,W], ``g_acc`` and ``g_depth`` [V,H,W] twice: as the default backward's
    atomics sum them, and (keys ending in ``_det``) as the deterministic backward's fixed point does.  Images planar.
    Also the masks ``wide_pairs`` [V,n] (a decision undecided), ``wide_points`` [n] (a point gradient that sums such a
    pair), ``wide_pixels`` [V,5,H,W] (rendering-gradient elements such a pair reaches), ``inf_pairs`` [V,n] (an
    infinite bound), and ``max_terms``, the most terms one rendering-gradient element sums."""
    pts = _f64(points).reshape(-1, 3)
    w2 = _f64(w2cs).reshape(-1, 4, 4)
    kk = _f64(ixts).reshape(-1, 3, 3)
    ref, img, ac, dp = _f64(img_ref), _f64(image), _f64(acc), _f64(depth)
    V, _, H, W = ref.shape
    n = pts.shape[0]
    HW = H * W
    stack = np.concatenate([ref.reshape(V, 3, HW), img.reshape(V, 3, HW), ac.reshape(V, 1, HW), dp.reshape(V, 1, HW)], 1)
    g = None if g_feats is None else _f32(g_feats).reshape(V, 8, n).astype(np.float64)
    fv, fe = np.zeros((V, 8, n)), np.zeros((V, 8, n))
    gp = [[] for _ in range(3)]
    rv, re_, rm, rabs = (np.zeros((V, 5, HW)) for _ in range(4))
    wide_pix = np.zeros((V, 5, HW), bool)
    wide_pairs, inf_pairs = np.zeros((V, n), bool), np.zeros((V, n), bool)
    for v in range(V if n else 0):       # no point: nothing sampled, every gradient 0
        vw = _View(pts, w2[v], kk[v], W, H)
        E, Km = w2[v], kk[v]
        inf_pairs[v] = vw.inf
        und_xy = vw.ax["und"] | vw.ay["und"]
        # sign of d over the box, then the evaluations: decided pairs at the 4 corners of their cell, the others at
        # every side
        allidx = np.arange(n)
        d = _Hull()
        for sub, u in ((allidx[~und_xy], False), (allidx[und_xy], True)):
            if sub.size == 0:
                continue
            r = _eval(stack[v], vw, sub, _positions(vw.ax, sub, u), _positions(vw.ay, sub, u), [1.0], None, W, H,
                      False, Km, E, only_d=True)["d"]
            if d.lo is None:
                d.lo, d.hi, d.r = (np.zeros(n) for _ in range(3))
            d.lo[sub], d.hi[sub], d.r[sub] = r.lo, r.hi, r.r
        smin, smax = _sign_set(d)
        und = und_xy | (smin != smax)
        wide_pairs[v] = und
        res = {}
        for sub, u in ((allidx[~und], False), (allidx[und], True)):
            if sub.size == 0:
                continue
            signs = [smin[sub]] if not u else [smin[sub], smax[sub]]
            res[u] = (sub, _eval(stack[v], vw, sub, _positions(vw.ax, sub, u), _positions(vw.ay, sub, u), signs, g[v]
                                 if g is not None else None, W, H, g is not None, Km, E))
        # the centre: float64 decisions at the float64 coordinates (the value of a decided element)
        c0x, c0y = vw.ax["c0"], vw.ay["c0"]
        dcen = _eval(stack[v], vw, allidx, [(c0x, np.clip(vw.ax["v"], c0x, c0x + 1))],
                     [(c0y, np.clip(vw.ay["v"], c0y, c0y + 1))], [None], None, W, H, False, Km, E, only_d=True)["d"]
        s0 = np.sign(dcen.lo)
        cen = _eval(stack[v], vw, allidx, [(c0x, np.clip(vw.ax["v"], c0x, c0x + 1))],
                    [(c0y, np.clip(vw.ay["v"], c0y, c0y + 1))], [s0], g[v] if g is not None else None, W, H,
                    g is not None, Km, E)

        def combine(key, k):
            """(value, bound) over all pairs: decided -> the centre value with the corners' largest distance from it,
            widened -> the hull's midpoint with its half-range."""
            val, err = np.zeros(n), np.zeros(n)
            for u, (sub, r) in res.items():
                h = r[key][k]
                c = cen[key][k].lo[sub]
                if u:
                    val[sub] = 0.5 * (h.lo + h.hi)
                    err[sub] = 0.5 * (h.hi - h.lo) + h.r
                else:
                    val[sub] = c
                    err[sub] = np.maximum(h.hi - c, c - h.lo) + np.maximum(h.r, cen[key][k].r[sub])
            return val, err

        for c in range(8):
            fv[v, c], fe[v, c] = combine("feats", c)
        fe[v][:, vw.inf] = np.inf
        if g is None:
            continue
        for k in range(3):
            a, b = combine("grad", k)
            gp[k].append(EB(a, np.where(vw.inf, np.inf, b)))
        # rendering gradients: per (pair, slot) the tap weight's hull, times each channel's upstream
        st = stencil(vw, W, H, und)
        for u in (False, True):
            for s_ in range(9):
                i = np.nonzero(st["touched"][s_] & (und == u))[0]
                if i.size == 0:
                    continue
                wv, wd, wr = st["v"][s_, i], st["d"][s_, i], st["r"][s_, i]
                pix = (st["Y"][s_, i] * W + st["X"][s_, i]).astype(np.int64)
                for c in range(3, 8):
                    go = g[v, c, i]
                    if c < 7:
                        tv = go * wv
                        te = np.abs(go) * (wd + wr) + U * np.abs(go) * (np.abs(wv) + wd + wr)
                    else:
                        lo_s, hi_s = smin[i], smax[i]
                        cands = [g[v, 7, i] * s * wx for s in (lo_s, hi_s) for wx in (wv - wd - wr, wv + wd + wr)]
                        tlo, thi = np.minimum.reduce(cands), np.maximum.reduce(cands)
                        dec = lo_s == hi_s
                        tv = np.where(dec, g[v, 7, i] * lo_s * wv, 0.5 * (tlo + thi))
                        big = np.maximum(np.abs(tlo), np.abs(thi))
                        te = np.where(dec, np.abs(g[v, 7, i]) * (wd + wr) + U * np.abs(g[v, 7, i]) * (np.abs(wv) + wd + wr),
                                      0.5 * (thi - tlo) + U * big)
                    ch = c - 3
                    rv[v, ch] += np.bincount(pix, tv, HW)
                    re_[v, ch] += np.bincount(pix, te, HW)
                    rabs[v, ch] += np.bincount(pix, np.abs(tv) + te, HW)
                    rm[v, ch] += np.bincount(pix, minlength=HW)
                    if u:
                        wide_pix[v, ch, np.unique(pix)] = True
        if vw.inf.any():
            re_[v] = np.inf
    out = {"feats": EB(fv, fe), "wide_pairs": wide_pairs, "inf_pairs": inf_pairs, "wide_points": wide_pairs.any(0)}
    if g is None:
        return out
    # the sum over the views, in any order
    g_points = [sum_any_order(gp[k]) if n else EB(np.zeros(0)) for k in range(3)]
    out["g_points"] = EB(np.stack([x.v for x in g_points], 1), np.stack([x.e for x in g_points], 1))
    gam = np.maximum(rm - 1, 0) * U
    L = ceil_log2(4 * V * n)
    k = scale_exp(abs_bits_max(g_feats), L)
    fixed = re_ + rm * 2.0 ** -(k + 1)
    for sfx, e in (("", re_ + gam / (1 - gam) * rabs), ("_det", fixed + U * (np.abs(rv) + fixed) + SUB_ULP)):
        e = np.where(rm > 0, e, 0.0)
        out["g_image" + sfx] = EB(rv[:, :3].reshape(V, 3, H, W), e[:, :3].reshape(V, 3, H, W))
        out["g_acc" + sfx] = EB(rv[:, 3].reshape(V, H, W), e[:, 3].reshape(V, H, W))
        out["g_depth" + sfx] = EB(rv[:, 4].reshape(V, H, W), e[:, 4].reshape(V, H, W))
    out["wide_pixels"] = wide_pix.reshape(V, 5, H, W)
    out["max_terms"] = int(rm.max()) if rm.size else 0
    return out


# ------------------------------------------------------------------------------------- det_sum.cuh, restated on the host

def _f32(a):
    if hasattr(a, "detach"):
        a = a.detach().cpu().numpy()
    return np.ascontiguousarray(a, dtype=np.float32)


def ceil_log2(n: int) -> int:
    return 0 if n <= 1 else int(n - 1).bit_length()


def abs_bits_max(g) -> int:
    a = _f32(g).reshape(-1)
    return int((a.view(np.uint32) & np.uint32(0x7FFFFFFF)).max()) if a.size else 0


def scale_exp(bound_bits: int, L: int) -> int:
    e = bound_bits >> 23
    return (K_SUM_BITS - 1) - L - ((1 if e == 0 else e) - 126)
