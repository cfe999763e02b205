"""Float64 statement, with a bound per element, of the fused MS-SSIM term (lara_b200/csrc/ms_ssim.cu).

TEST INFRASTRUCTURE ONLY -- importable from tests/; never from lara_b200/.

Every value is an ``oracle.EB``: the float64 value of ``ms_ssim.cu``'s formulas, in its order of operations (not the
library's fp32 op sequence), with a bound on how far the kernel's fp32 evaluation may lie from it.  Decisions (relu
per plane) are taken from the bounds, as ``chain64`` takes them from the fp32 inputs.  The rules:

* **Window.** The 11 fp32 taps are exact constants: they are the contract (DESIGN §3.12).  ``window()`` builds them
  as ``level_args`` does; the suite checks them bit for bit against the library's ``_fspecial_gauss_1d``.  C1 and C2
  are the float64 ``(K data_range)^2`` with half an ulp for their rounding to fp32 (``EB.w``).
* **Correctly rounded operations** (no ``--use_fast_math``: ``/`` is IEEE): an operation whose exact result on the
  exact operands is ``v`` and on the computed operands lies within ``e`` of ``v`` returns ``e + U (|v| + e)``,
  ``U = 2^-24`` (half an ulp of the result, ``chain64._rn``), plus half a subnormal spacing.  A product inside an
  ``fmaf`` is exact; ``u * u`` and ``u * v`` before it are rounded once.  nvcc's contraction of ``a * b + c`` into one
  ``fmaf`` drops a rounding, so the bound covers either form.  Scaling by 2 or 0.25 is exact.
* **11-tap fma chains** -- the forward's H then W passes of ``x, y, x^2, y^2, xy``, the backward's recomputation of
  the same passes (identical operations, so the same values) and its two G^T passes: ``s_t = fmaf(g_t, u_t, s_{t-1})``
  in the kernel's tap order ``t = 0..10``.  The bound is what the inputs bring in, ``sum g_t e_t``, plus half an ulp of
  every running sum, ``U sum_t |s_t|`` (with the running bound inside, as above).  EB's default rule would be a full
  ulp per operation and an order-independent ``11 K sum |g_t u_t|``, three to four times looser.
* **Pooling.** Three fp32 additions in the kernel's order (row 0 left, row 0 right, row 1 left, row 1 right), then an
  exact ``* 0.25``; the zero padding is an exact operand and counts in the divisor.
* **Maps.** ``sigma = G(..) - mu mu``: the cancellation is real and the bound carries it (the bound of ``G(xx)`` is
  relative to ``G(xx)``, not to ``sigma``).  Then ``cs``, the level-4 ``ssim``, and the backward's ``rd = 1 / dcs``,
  ``cmu, cxx, cxy``, ``lum, lmu`` and ``A, B, C`` as ``ms_ssim.cu`` writes them.
* **Means.** fp64 sums of the fp32 map values: the sum of the element bounds divided by the count, plus ``2 n 2^-53``
  of the sum of magnitudes for any order of ``n`` double additions.  This bound is a worst case summed over every
  pixel of the level and inherently loose (typically 1e-3 relative while the kernel's mean is ~1e-8 from float64); it
  does not catch small errors in the means.
* **Finalize.** A plane with ``|m_l| <= e_l`` at any level is *undecided* (excluded, like the blend replay's band
  Gaussians; every test case asserts it has none).  ``v = prod m_l^w_l`` in double is bounded by evaluating it at
  ``m_l +- e_l`` (it is monotone in each ``m_l``), not to first order; ``coef_l = fp32(w_l v / m_l scale / count_l)``
  likewise (increasing in ``m_j``, j != l, decreasing in ``m_l``), plus its rounding to fp32.  The result is a double
  mean of ``v`` and one rounding to fp32.  A plane decided non-positive has value 0 and coefficients exactly 0.
* **Backward per level.** ``k = fp32(coef) * fp32(upstream)`` rounded once; ``dX_l = fmaf(2x, G^T B, G^T A)``, then
  ``fmaf(y, G^T C, .)``, then ``+ 0.25 dX_{l+1}[parent]`` with parent ``((y + py) / 2, (x + px) / 2)``.  A plane whose
  coefficient is decided 0 gives exactly ``0.25 dX_{l+1}[parent]`` (0 at level 4), with only that term's bound.

Two forms.  ``ms_ssim64(X, Y, ...)`` is end to end from the fp32 level-0 X and Y: every later quantity inherits the
bounds before it, and through ``k`` the loose means, so each gradient element's bound has a floor of about 1e-3 of its
value.  ``ms_ssim64(X, Y, ..., state=...)`` is link by link, each on the kernel's own fp32 inputs (the workspace, as
``lara_b200.debug.unpack_ms_ssim`` reads it): ``X_l, Y_l`` from the kernel's ``X_{l-1}, Y_{l-1}``; the value and the
coefficients from the kernel's fp64 means (double arithmetic and one fp32 rounding: tight); ``dX_l`` from the kernel's
``X_l, Y_l``, its coefficient and its ``dX_{l+1}``.  A wrong level-4 gradient shows in ``dX_4`` directly rather than after
its division by 256 into a level-0 pixel.

``arith=F32`` runs the same sequence as an fp32 NumPy emulation of the kernel (each ``fmaf`` a float64 operation
rounded to fp32, the double parts in double): the suite checks that it lies within the bounds.
"""
from __future__ import annotations

import numpy as np

from .oracle import EB

U = 2.0 ** -24                  # half an ulp, relative: one correctly rounded fp32 operation
SUB = 2.0 ** -150               # half the spacing of fp32's subnormals
D = 2.0 ** -53                  # half a double ulp, relative
WEIGHTS = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333)
LEVELS = 5
R = 10                          # window size - 1
f32, f64 = np.float32, np.float64


def window() -> np.ndarray:
    """ms_ssim.cu's fp32 taps: exp(-(i - 5)^2 / 4.5f) rounded to fp32, their double sum rounded once, fp32 division."""
    c = (np.arange(11) - 5).astype(f32)
    e = np.exp((-(c * c) / f32(4.5)).astype(f64)).astype(f32)
    return (e / f32(e.astype(f64).sum())).astype(f32)


def _rn(v, e) -> EB:
    """One correctly rounded fp32 operation (module docstring)."""
    return EB(v, e + U * (np.abs(v) + e) + SUB)


def _take(a: np.ndarray, axis: int, start: int, n: int) -> np.ndarray:
    sl = [slice(None)] * a.ndim
    sl[axis] = slice(start, start + n)
    return a[tuple(sl)]


def _pad(a: np.ndarray, axis: int, lo: int, hi: int) -> np.ndarray:
    p = [(0, 0)] * a.ndim
    p[axis] = (lo, hi)
    return np.pad(a, p)


class Bound:
    """Float64 values with the bound of the kernel's fp32 evaluation (EB)."""
    exact = staticmethod(lambda a: EB(np.asarray(a, f64)))
    const = staticmethod(lambda c: EB.w(float(c)))

    @staticmethod
    def mul(a, b):
        a, b = EB.w(a), EB.w(b)
        return _rn(a.v * b.v, np.abs(a.v) * b.e + np.abs(b.v) * a.e + a.e * b.e)

    @staticmethod
    def add(a, b):
        a, b = EB.w(a), EB.w(b)
        return _rn(a.v + b.v, a.e + b.e)

    @staticmethod
    def sub(a, b):
        a, b = EB.w(a), EB.w(b)
        return _rn(a.v - b.v, a.e + b.e)

    @staticmethod
    def div(a, b):
        a, b = EB.w(a), EB.w(b)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = a.v / b.v
            den = np.abs(b.v) - b.e
            e = np.where(den > 0, (a.e + np.abs(v) * b.e) / np.where(den > 0, den, 1.0), np.inf)
        return _rn(v, e)

    @staticmethod
    def fma(a, b, c):
        a, b, c = EB.w(a), EB.w(b), EB.w(c)
        return _rn(a.v * b.v + c.v, np.abs(a.v) * b.e + np.abs(b.v) * a.e + a.e * b.e + c.e)

    @staticmethod
    def scale(a, s):                    # by a power of two: exact
        return EB(a.v * s, a.e * abs(s))

    @staticmethod
    def neg(a):
        return EB(-a.v, a.e)

    @staticmethod
    def pad(a, axis, lo, hi):
        return EB(_pad(a.v, axis, lo, hi), _pad(a.e, axis, lo, hi))

    @staticmethod
    def index(a, iy, ix):
        return EB(a.v[..., iy[:, None], ix[None, :]], a.e[..., iy[:, None], ix[None, :]])

    @staticmethod
    def where(m, a, b):
        return EB.where(m, a, b)

    @staticmethod
    def chain(u: EB, g, axis, offs, n) -> EB:
        """s_t = fmaf(g_t, u[i + offs[t]], s_{t-1}) along `axis`, n outputs."""
        shape = list(u.v.shape)
        shape[axis] = n
        sv, se, t = np.zeros(shape), np.zeros(shape), np.empty(shape)
        for gt, o in zip(g.astype(f64), offs):
            sv += gt * _take(u.v, axis, o, n)
            se += gt * _take(u.e, axis, o, n)
            np.abs(sv, out=t)
            t += se
            t *= U
            se += t
            se += SUB
        return EB(sv, se)


class F32:
    """The fp32 emulation of the kernel's sequence: numpy's float32 operations are correctly rounded; an fmaf is a
    float64 operation rounded to fp32."""
    exact = staticmethod(lambda a: np.asarray(a, f32))
    const = staticmethod(lambda c: f32(c))
    mul = staticmethod(lambda a, b: (f32(a) * f32(b)) if np.isscalar(a) and np.isscalar(b) else
                       np.multiply(a, b, dtype=f32))
    add = staticmethod(lambda a, b: np.add(a, b, dtype=f32))
    sub = staticmethod(lambda a, b: np.subtract(a, b, dtype=f32))
    div = staticmethod(lambda a, b: np.divide(a, b, dtype=f32))
    fma = staticmethod(lambda a, b, c: (np.asarray(a, f64) * np.asarray(b, f64) + np.asarray(c, f64)).astype(f32))
    scale = staticmethod(lambda a, s: np.multiply(a, f32(s), dtype=f32))
    neg = staticmethod(lambda a: -a)
    pad = staticmethod(_pad)
    index = staticmethod(lambda a, iy, ix: a[..., iy[:, None], ix[None, :]])
    where = staticmethod(lambda m, a, b: np.where(m, a, b).astype(f32))

    @staticmethod
    def chain(u, g, axis, offs, n):
        shape = list(u.shape)
        shape[axis] = n
        s = np.zeros(shape, f64)
        for gt, o in zip(g.astype(f64), offs):
            s = (gt * _take(u, axis, o, n).astype(f64) + s).astype(f32).astype(f64)
        return s.astype(f32)


def _val(a):
    return a.v if isinstance(a, EB) else np.asarray(a, f64)


# ------------------------------------------------------------------------------------------------------- one level

def pool(A, x):
    """X_{l+1} of one plane: avg_pool2d(2, padding=s % 2) as the forward kernel sums a cell."""
    H, W = _val(x).shape[-2:]
    py, px = H % 2, W % 2
    p = A.pad(A.pad(x, -2, py, py), -1, px, px)
    h, w = (H + 2 * py) // 2, (W + 2 * px) // 2
    q = lambda dy, dx: _sub2(p, dy, dx, h, w)       # noqa: E731
    t = A.add(q(0, 0), q(0, 1))
    t = A.add(t, q(1, 0))
    t = A.add(t, q(1, 1))
    return A.scale(t, 0.25)


def _sub2(p, dy, dx, h, w):
    if isinstance(p, EB):
        return EB(p.v[dy:dy + 2 * h:2, dx:dx + 2 * w:2], p.e[dy:dy + 2 * h:2, dx:dx + 2 * w:2])
    return p[dy:dy + 2 * h:2, dx:dx + 2 * w:2]


def level_maps(A, x, y, g, c1, c2, last):
    """The filtered maps of one plane at one level on the valid outputs [h - 10, w - 10], and its mean's input (cs, or
    the ssim map at level 4)."""
    H, W = _val(x).shape[-2:]
    q = (x, y, A.mul(x, x), A.mul(y, y), A.mul(x, y))
    f = [A.chain(A.chain(u, g, -2, range(R + 1), H - R), g, -1, range(R + 1), W - R) for u in q]
    mx, my = f[0], f[1]
    mxx, myy, mxy = A.mul(mx, mx), A.mul(my, my), A.mul(mx, my)
    sx, sy, sxy = A.sub(f[2], mxx), A.sub(f[3], myy), A.sub(f[4], mxy)
    dcs = A.add(A.add(sx, sy), c2)
    cs = A.div(A.add(A.scale(sxy, 2.0), c2), dcs)
    m = dict(mx=mx, my=my, mxx=mxx, myy=myy, mxy=mxy, dcs=dcs, cs=cs, term=cs)
    if last:
        dl = A.add(A.add(mxx, myy), c1)
        lum = A.div(A.add(A.scale(mxy, 2.0), c1), dl)
        m.update(dl=dl, lum=lum, term=A.mul(lum, cs))
    return m


def level_grad(A, x, y, maps, g, k, gnext, px, py, last):
    """dX_l of one plane: the coefficient maps on the valid outputs, G^T along y then x (taps in the kernel's gather
    order), the three fmaf and the pooling backward.  k: the plane's fp32 coef * upstream (None: decided 0)."""
    H, W = _val(x).shape[-2:]
    if gnext is not None:
        iy, ix = (np.arange(H) + py) // 2, (np.arange(W) + px) // 2
        parent = A.scale(A.index(gnext, iy, ix), 0.25)
    if k is None:                                   # the kernel skips everything but the pooling term
        return parent if gnext is not None else A.exact(np.zeros((H, W)))
    rel = 0.0
    if isinstance(k, EB) and float(k.e) > 0:
        # everything below is linear in k, bounds included: an error of k is one factor (1 + rel) on the level's own
        # term, not an independent error of each of the terms that cancel in it
        rel = float(k.e) / abs(float(k.v))
        k = EB(k.v)
    mx, my, cs, dcs = maps["mx"], maps["my"], maps["cs"], maps["dcs"]
    rd = A.div(1.0, dcs)
    cmu = A.mul(A.scale(A.sub(A.mul(mx, cs), my), 2.0), rd)
    cxx = A.mul(A.neg(cs), rd)
    cxy = A.scale(rd, 2.0)
    if last:
        lum, dl = maps["lum"], maps["dl"]
        lmu = A.div(A.scale(A.sub(my, A.mul(mx, lum)), 2.0), dl)
        kl = A.mul(k, lum)
        cm = (A.mul(k, A.add(A.mul(cs, lmu), A.mul(lum, cmu))), A.mul(kl, cxx), A.mul(kl, cxy))
    else:
        cm = (A.mul(k, cmu), A.mul(k, cxx), A.mul(k, cxy))
    gt = []
    for a in cm:                                    # input row y gathers output rows y - t: padded offset R - t
        t = A.chain(A.pad(a, -2, R, R), g, -2, [R - t for t in range(R + 1)], H)
        gt.append(A.chain(A.pad(t, -1, R, R), g, -1, [R - t for t in range(R + 1)], W))
    d = A.fma(A.scale(x, 2.0), gt[1], gt[0])
    d = A.fma(y, gt[2], d)
    if rel:
        d = EB(d.v, d.e * (1 + rel) + rel * np.abs(d.v))
    if gnext is not None:
        d = A.add(d, parent)
    return d


# ----------------------------------------------------------------------------------------------- means and finalize

def mean_bound(term: EB):
    """A level's mean of one plane: (value, bound) of the kernel's fp64 sum of its fp32 map over the count."""
    n = term.v.size
    mag = float(np.abs(term.v).sum() + term.e.sum())
    v = float(term.v.sum()) / n
    return v, (float(term.e.sum()) + 2 * n * D * mag) / n + 2 * D * abs(v)


def finalize(m, e, scale, count):
    """value and coefficients of one plane from its five means m (bounds e): Bound form.  Returns (state, val (v, e),
    coef [(v, e)] * 5) with state "pos", "zero" (decided non-positive) or "undecided"."""
    m, e = np.asarray(m, f64), np.asarray(e, f64)
    if (np.abs(m) <= e).any():
        return "undecided", (0.0, np.inf), [(0.0, np.inf)] * LEVELS
    if (m < 0).any():
        return "zero", (0.0, 0.0), [(0.0, 0.0)] * LEVELS
    w = np.asarray(WEIGHTS)
    v = float(np.prod(m ** w))
    lo, hi = float(np.prod((m - e) ** w)), float(np.prod((m + e) ** w))
    val = (v, max(hi - v, v - lo) + 16 * D * v)
    coef = []
    for l in range(LEVELS):
        c = WEIGHTS[l] * v / m[l] * scale / count[l]
        mh, ml = m + e, m - e
        mh[l], ml[l] = m[l] - e[l], m[l] + e[l]
        ch = WEIGHTS[l] * float(np.prod(mh ** w)) / mh[l] * scale / count[l]
        cl = WEIGHTS[l] * float(np.prod(ml ** w)) / ml[l] * scale / count[l]
        ein = max(ch - c, c - cl) + 24 * D * c
        coef.append((c, ein + U * (abs(c) + ein) + SUB))
    return "pos", val, coef


def finalize32(m, scale, count):
    """ms_ssim_finalize_kernel on one plane, in double, the coefficients rounded to fp32."""
    if not all(mi > 0 for mi in m):
        return "zero", 0.0, [f32(0)] * LEVELS
    v = 1.0
    for l in range(LEVELS):
        v *= float(m[l]) ** WEIGHTS[l]
    return "pos", v, [f32(WEIGHTS[l] * v / m[l] * scale / count[l]) for l in range(LEVELS)]


# ----------------------------------------------------------------------------------------------------- the statement

def _consts(A, data_range):
    c1, c2 = 0.01 * float(f32(data_range)), 0.03 * float(f32(data_range))
    return A.const(c1 * c1), A.const(c2 * c2)


def plane64(A, x0, y0, g, c1, c2, scale, up, link=None, keep_maps=False):
    """One (b, c) plane through all five levels.  A = Bound or F32.  `link` (Bound only): the kernel's own per-plane
    state {"X": [l] (None at 0), "Y", "mean" [5], "coef" [5], "dX" [l] (None at 0)}: each link then starts from it.
    Returns {"X", "Y" (lists, level 0 the input), "m" [(v, e)] or doubles, "state", "val", "coef", "dX" (list),
    "maps" (term maps if keep_maps)}."""
    xs, ys = [A.exact(x0)], [A.exact(y0)]
    for l in range(1, LEVELS):
        px, py = (xs[-1], ys[-1]) if link is None else (A.exact(link["X"][l - 1] if l > 1 else x0),
                                                         A.exact(link["Y"][l - 1] if l > 1 else y0))
        xs.append(pool(A, px))
        ys.append(pool(A, py))
    ins = [(xs[l], ys[l]) if link is None or l == 0 else (A.exact(link["X"][l]), A.exact(link["Y"][l]))
           for l in range(LEVELS)]
    maps, means, count = [], [], []
    for l in range(LEVELS):
        mp = level_maps(A, ins[l][0], ins[l][1], g, c1, c2, l == LEVELS - 1)
        maps.append(mp)
        count.append(float(_val(mp["term"]).size))
        if A is Bound:
            means.append(mean_bound(mp["term"]))
        else:
            means.append(float(mp["term"].astype(f64).sum()) / mp["term"].size)
    if A is Bound:
        fm = [mm[0] for mm in means] if link is None else [float(v) for v in link["mean"]]
        fe = [mm[1] for mm in means] if link is None else [0.0] * LEVELS
        st, val, coef = finalize(fm, fe, scale, count)
        ks = [None if st != "pos" else _rn(coef[l][0] * float(up), abs(float(up)) * coef[l][1]) for l in range(LEVELS)]
        if link is not None and st == "pos":
            ks = [_rn(float(f32(link["coef"][l])) * float(up), 0.0) for l in range(LEVELS)]
    else:
        st, val, coef = finalize32(means, scale, count)
        ks = [None if st != "pos" else f32(coef[l]) * f32(up) for l in range(LEVELS)]
    dX = [None] * LEVELS
    for l in range(LEVELS - 1, -1, -1):
        last = l == LEVELS - 1
        gnext = None if last else (dX[l + 1] if link is None else A.exact(link["dX"][l + 1]))
        H, W = _val(ins[l][0]).shape
        dX[l] = level_grad(A, ins[l][0], ins[l][1], maps[l], g, ks[l], gnext, W % 2 if not last else 0,
                           H % 2 if not last else 0, last)
        if not keep_maps:
            maps[l] = None
    return dict(X=xs, Y=ys, m=means, state=st, val=val, coef=coef, dX=dX,
                maps=[None if mp is None else mp["term"] for mp in maps])


def ms_ssim64(X, Y, data_range=1.0, size_average=True, upstream=None, state=None, arith=Bound, keep_maps=False,
              planes=None):
    """The statement on fp32 logical images X, Y [B,C,H,W].  upstream: fp32 [1] or [B] (default ones).  state: the
    kernel's workspace as numpy ({"X", "Y", "dX": lists over levels of [B,C,h,w] (None at 0), "mean" [5,B,C],
    "coef" [5,B,C]}) for the link-by-link form.  planes: iterate only over these (b, c).  Returns
    {"planes": {(b, c): plane64's dict}, "out": (v, e) per output (Bound) or doubles (F32)}."""
    X, Y = np.asarray(X, f32), np.asarray(Y, f32)
    B, C = X.shape[:2]
    P = B * C
    up = np.ones(1 if size_average else B, f32) if upstream is None else np.asarray(upstream, f32).reshape(-1)
    g = window()
    c1, c2 = _consts(arith, data_range)
    scale = 1.0 / (P if size_average else C)
    res = {}
    for b in range(B):
        for c in range(C):
            if planes is not None and (b, c) not in planes:
                continue
            link = None
            if state is not None:
                link = {k: [None if a is None else a[b, c] for a in state[k]] for k in ("X", "Y", "dX")}
                link["mean"], link["coef"] = state["mean"][:, b, c], state["coef"][:, b, c]
            res[(b, c)] = plane64(arith, X[b, c], Y[b, c], g, c1, c2, scale, up[0 if size_average else b], link,
                                  keep_maps)
    out = None
    if planes is None:
        groups = [[(b, c) for b in range(B) for c in range(C)]] if size_average else \
            [[(b, c) for c in range(C)] for b in range(B)]
        out = []
        for grp in groups:
            if arith is Bound:
                v = sum(res[p]["val"][0] for p in grp) / len(grp)
                e = sum(res[p]["val"][1] for p in grp) / len(grp) + 2 * len(grp) * D * abs(v)
                out.append((v, e + U * (abs(v) + e)))
            else:
                out.append(float(f32(sum(res[p]["val"] for p in grp) / len(grp))))
    return {"planes": res, "out": out}
