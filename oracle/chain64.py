"""Float64 statements, with a bound per element, of the kernels around the rasterizer in LaRa's training step: the fused
``render_img`` epilogue (lara_b200/csrc/epilogue.cu), the loss producer (csrc/loss.cu) and the decoder layout
(csrc/decoder.cu).

TEST INFRASTRUCTURE ONLY -- importable from tests/; never from lara_b200/.

Every value is an ``oracle.EB``: the float64 value of the kernel's formula together with a bound on what any fp32
evaluation of the same formula may differ by (the per-operation rules of the blend replay, oracle/surfel_oracle.c).
Decisions are taken from the fp32 inputs, as the blend replay takes the forward's decisions: the clamp masks, and
whether ``fp32(D) / fp32(alpha)`` and the median depth are finite (numpy's float32 division is correctly rounded, like
the kernel's ``/`` without ``--use_fast_math``).  Two more rules are added here:

* fp32's range (``_ovf``): an fp32 evaluation overflows where the value plus its bound exceeds FLT_MAX, and the bound is
  then infinite; below FLT_MIN an inexact value carries the absolute error of gradual underflow.  The rule is applied to
  every result and to each intermediate that can leave the range on its own: the points, their differences, the cross
  product and its squared norm, ``g * alpha`` and ``(D / alpha) / alpha``.  The other intermediates (the four-neighbour
  terms, ``n . G``, the loss and decoder products) are checked at the result only: an fp32 overflow or underflow inside
  them whose result is back in range is not modelled, so the bound is claimed only where they stay in range;
* ``F.normalize``'s ``max(norm, 1e-12)``: where ``|norm - 1e-12|`` lies within norm's bound the branch is not decided
  by the inputs -- a *band* element, excluded like the blend replay's band Gaussians.  Where the cross product's bound
  reaches ``|c|`` the normalisation's division already returns an infinite bound.
"""
from __future__ import annotations

import numpy as np

from .oracle import EB, K

FLT_MAX = float(np.finfo(np.float32).max)
FLT_MIN = float(np.finfo(np.float32).tiny)
SUB_ULP = 2.0 ** -149           # the spacing of fp32's subnormals
EPS = 1e-12                     # F.normalize's eps; the kernel's 1e-12f and 1e12f are its fp32 roundings (EB.w)
_D = 2.0 ** -52                 # one double ulp, relative: the loss kernels' double sums


def _ovf(x: EB) -> EB:
    """fp32's range: an infinite bound where an fp32 evaluation may overflow (or the value is not finite), and below
    FLT_MIN the absolute error of gradual underflow (half a subnormal ulp per operation, for up to eight) unless the
    value is exact."""
    with np.errstate(invalid="ignore"):
        bad = ~(np.abs(x.v) + x.e <= FLT_MAX)
        tiny = (np.abs(x.v) - x.e < FLT_MIN) & ~((x.e == 0) & (x.v.astype(np.float32).astype(np.float64) == x.v))
    return EB(x.v, np.where(bad, np.inf, x.e + np.where(tiny, 4 * SUB_ULP, 0.0)))


def _exact(s: EB, a: EB, b: EB) -> EB:
    """No rounding where both operands are exact and the float64 result is an fp32 value: o + 0 * d at an empty pixel,
    the difference of two such points, 1 - depth_ratio, a median times depth_ratio = 1."""
    exact = (a.e == 0) & (b.e == 0) & (s.v.astype(np.float32).astype(np.float64) == s.v)
    return EB(s.v, np.where(exact, 0.0, s.e))


def _add(a, b) -> EB:
    a, b = EB.w(a), EB.w(b)
    return _exact(a + b, a, b)


def _mul(a, b) -> EB:
    a, b = EB.w(a), EB.w(b)
    return _exact(a * b, a, b)


def _clean(x: EB) -> EB:
    """A NaN bound (0 * inf inside a product) is an unknown one: infinite."""
    return EB(x.v, np.where(np.isnan(x.e), np.inf, x.e))


def _f32(a) -> np.ndarray:
    if hasattr(a, "detach"):
        a = a.detach().cpu().numpy()
    return np.asarray(a, dtype=np.float32)


def _nan_to_num32(v32: np.ndarray) -> np.ndarray:
    """torch.nan_to_num(v, nan=0, posinf=0) on fp32: -inf -> the lowest finite float."""
    out = np.where(np.isnan(v32) | (v32 == np.inf), np.float32(0), v32)
    return np.where(out == -np.inf, np.float32(-FLT_MAX), out).astype(np.float32)


# ------------------------------------------------------------------------------------------------------------ epilogue

class EpilogueState:
    """The epilogue forward of one view: inputs as float64, the fp32 decisions, and the intermediate EB values the
    vjp reuses."""

    def __init__(self, color, allmap, rays, viewmatrix, depth_ratio):
        c32, a32 = _f32(color), _f32(allmap)
        self.H, self.W = c32.shape[1], c32.shape[2]
        self.color = c32.astype(np.float64)
        self.allmap = a32.astype(np.float64)
        self.rays = None if rays is None else _f32(rays).astype(np.float64)
        self.vm = _f32(viewmatrix).reshape(16).astype(np.float64)
        self.r = float(np.float32(depth_ratio))          # passed to the kernel as a float
        D32, al32, med32 = a32[0], a32[1], a32[5]
        with np.errstate(divide="ignore", invalid="ignore"):
            q32 = D32 / al32
        self.q_ok = np.isfinite(q32)
        self.m_ok = np.isfinite(med32)
        # nan_to_num of the fp32 quotient: where it is finite the float64 quotient with its bound, else what
        # nan_to_num makes of the non-finite fp32 value (exact)
        D, al = EB(self.allmap[0]), EB(self.allmap[1])
        with np.errstate(divide="ignore", invalid="ignore"):
            q = D / EB(np.where(self.q_ok, al.v, 1.0))
        self.dexp = EB(np.where(self.q_ok, q.v, _nan_to_num32(q32)), np.where(self.q_ok, q.e, 0.0))
        self.dmed = EB(_nan_to_num32(med32).astype(np.float64))
        r = self.r
        self.one_m = _add(1.0, -EB.w(r))
        self.surf = _ovf(_add(_mul(self.dexp, self.one_m), _mul(r, self.dmed)))
        if self.rays is None:
            self.c = None
            return
        # back-projected points, then the central differences and the cross product at every interior pixel
        o = [EB(self.rays[..., k]) for k in range(3)]
        d = [EB(self.rays[..., 3 + k]) for k in range(3)]
        self.dir = d
        self.p = [_ovf(_add(o[k], self.surf * d[k])) for k in range(3)]
        H, W = self.H, self.W
        self.interior = np.zeros((H, W), bool)
        self.interior[1:-1, 1:-1] = True
        sl = lambda x, ys, xs: EB(np.pad(x.v[ys, xs], 1), np.pad(x.e[ys, xs], 1))     # noqa: E731 (zero border)
        if H >= 3 and W >= 3:
            self.dx = [_ovf(_add(sl(pk, slice(2, None), slice(1, -1)), -sl(pk, slice(None, -2), slice(1, -1))))
                       for pk in self.p]
            self.dy = [_ovf(_add(sl(pk, slice(1, -1), slice(2, None)), -sl(pk, slice(1, -1), slice(None, -2))))
                       for pk in self.p]
        else:
            z = EB(np.zeros((H, W)))
            self.dx, self.dy = [z, z, z], [z, z, z]
        dx, dy = self.dx, self.dy
        self.c = [_ovf(dx[1] * dy[2] - dx[2] * dy[1]), _ovf(dx[2] * dy[0] - dx[0] * dy[2]),
                  _ovf(dx[0] * dy[1] - dx[1] * dy[0])]
        c = self.c
        self.norm = _ovf(_ovf(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]).sqrt())
        # an infinite bound is not a band: the division by the norm then carries it into the result
        fin = np.isfinite(self.norm.e)
        with np.errstate(invalid="ignore"):
            self.band = self.interior & fin & ~(np.abs(self.norm.v - EPS) > self.norm.e)
        self.big = self.interior & ((self.norm.v > EPS) | ~fin) & ~self.band


def _rot(vm, n, transpose):
    """(n^T @ vm[:3,:3].T)_j = sum_i vm[4j+i] n_i (forward); the vjp sums vm[4i+j] g_i."""
    idx = (lambda j, i: 4 * i + j) if transpose else (lambda j, i: 4 * j + i)
    return [n[0] * EB.w(vm[idx(j, 0)]) + n[1] * EB.w(vm[idx(j, 1)]) + n[2] * EB.w(vm[idx(j, 2)]) for j in range(3)]


def epilogue64(color, allmap, rays, viewmatrix, depth_ratio, state: EpilogueState = None):
    """The six outputs of ``render_img_epilogue_torch``, planar: {name: EB} with image [3,H,W], depth [H,W],
    acc_map [H,W], rend_normal [3,H,W], depth_normal [3,H,W], rend_dist [H,W]; plus the band mask [H,W] and
    the mask of pixels whose depth_normal has an infinite bound."""
    s = state or EpilogueState(color, allmap, rays, viewmatrix, depth_ratio)
    H, W = s.H, s.W
    out = {"image": EB(np.clip(s.color, 0.0, 1.0)), "depth": s.surf, "acc_map": EB(s.allmap[1]),
           "rend_normal": _rot(s.vm, [EB(s.allmap[2 + k]) for k in range(3)], False), "rend_dist": EB(s.allmap[6])}
    out["rend_normal"] = EB(np.stack([x.v for x in out["rend_normal"]]), np.stack([x.e for x in out["rend_normal"]]))
    if s.c is None:
        out["depth_normal"] = EB(np.zeros((3, H, W)))
        return out, np.zeros((H, W), bool), np.zeros((H, W), bool)
    alpha = EB(s.allmap[1])
    length = EB.where(s.big, s.norm, EB.w(EPS))
    dn = []
    for k in range(3):
        with np.errstate(divide="ignore", invalid="ignore"):
            v = _clean(_ovf(s.c[k] / length * alpha))
        dn.append(EB(np.where(s.interior, v.v, 0.0), np.where(s.interior, v.e, 0.0)))
    out["depth_normal"] = EB(np.stack([x.v for x in dn]), np.stack([x.e for x in dn]))
    inf = s.interior & ~s.band & ~np.isfinite(out["depth_normal"].e).all(0)
    return out, s.band, inf


def epilogue_vjp64(color, allmap, rays, viewmatrix, depth_ratio, g_image=None, g_depth=None, g_acc=None,
                   g_rend_normal=None, g_depth_normal=None, g_rend_dist=None, state: EpilogueState = None):
    """dL/dcolor [3,H,W] and dL/dallmap [8,H,W] (EB) of the epilogue for planar upstreams ([3,H,W] / [H,W]; any may be
    None).  At alpha == 0 the D/alpha terms are 0 (the kernel's documented difference: torch's autograd gives NaN).
    Returns (d_color, d_allmap, excl [H,W]) with excl the pixels a band centre's gradient reaches (its four
    neighbours), which are not checked."""
    s = state or EpilogueState(color, allmap, rays, viewmatrix, depth_ratio)
    H, W = s.H, s.W
    z = np.zeros((H, W))
    up = lambda g, n: [EB(z)] * n if g is None else \
        [EB(_f32(g).reshape(n, H, W)[k].astype(np.float64)) for k in range(n)]        # noqa: E731
    gi, gd, ga, grn, gdn, gds = up(g_image, 3), up(g_depth, 1)[0], up(g_acc, 1)[0], up(g_rend_normal, 3), \
        up(g_depth_normal, 3), up(g_rend_dist, 1)[0]
    inside = (s.color >= 0.0) & (s.color <= 1.0)
    d_color = EB(np.where(inside, np.stack([x.v for x in gi]), 0.0))
    excl = np.zeros((H, W), bool)
    g_sd = gd
    if g_depth_normal is not None and s.c is not None:
        alpha = EB(s.allmap[1])
        G = [_ovf(gdn[k] * alpha) for k in range(3)]
        with np.errstate(divide="ignore", invalid="ignore"):
            inv = _clean(1.0 / EB.where(s.big, s.norm, 1.0))
            n = [_clean(s.c[k] * inv) for k in range(3)]
            nd = n[0] * G[0] + n[1] * G[1] + n[2] * G[2]
            gb = [_clean(_ovf((G[k] - n[k] * nd) * inv)) for k in range(3)]
        ge = [_ovf(G[k] * EB.w(1.0 / EPS)) for k in range(3)]
        gc = [EB.where(s.interior, EB.where(s.big, gb[k], ge[k]), 0.0) for k in range(3)]

        def shift(x: EB, dyy, dxx):
            """x at (y + dyy, x + dxx), zero outside the image."""
            v, e = np.zeros((H, W)), np.zeros((H, W))
            ys, yd = (slice(dyy, None), slice(None, H - dyy)) if dyy >= 0 else (slice(None, H + dyy), slice(-dyy, None))
            xs, xd = (slice(dxx, None), slice(None, W - dxx)) if dxx >= 0 else (slice(None, W + dxx), slice(-dxx, None))
            v[yd, xd], e[yd, xd] = x.v[ys, xs], x.e[ys, xs]
            return EB(v, e)

        def cross(u, w):
            return [u[1] * w[2] - u[2] * w[1], u[2] * w[0] - u[0] * w[2], u[0] * w[1] - u[1] * w[0]]
        # dL/dp of this pixel from the four centres whose differences it enters, in the kernel's order:
        # centre above (+ dy x gc), below (- dy x gc), left (+ gc x dx), right (- gc x dx)
        terms = []
        for (dyy, dxx, row, sign) in ((-1, 0, True, 1.0), (1, 0, True, -1.0), (0, -1, False, 1.0), (0, 1, False, -1.0)):
            g_c = [shift(gc[k], dyy, dxx) for k in range(3)]
            if row:
                t = cross([shift(s.dy[k], dyy, dxx) for k in range(3)], g_c)
            else:
                t = cross(g_c, [shift(s.dx[k], dyy, dxx) for k in range(3)])
            terms.append([_ovf(sign * t[k]) for k in range(3)])
        gp = [_ovf(terms[0][k] + terms[1][k] + terms[2][k] + terms[3][k]) for k in range(3)]
        g_sd = _clean(_ovf(gd + (gp[0] * s.dir[0] + gp[1] * s.dir[1] + gp[2] * s.dir[2])))
        b = s.band
        excl = np.zeros((H, W), bool)
        excl[:-1] |= b[1:]
        excl[1:] |= b[:-1]
        excl[:, :-1] |= b[:, 1:]
        excl[:, 1:] |= b[:, :-1]
    alpha = EB(s.allmap[1])
    g_exp = EB.where(s.q_ok, g_sd * s.one_m, 0.0)
    safe = EB(np.where(s.q_ok, alpha.v, 1.0))
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        d_D = _clean(_ovf(EB.where(s.q_ok, g_exp / safe, 0.0)))
        q = EB(np.where(s.q_ok, s.dexp.v, 0.0), np.where(s.q_ok, s.dexp.e, 0.0))
        d_al = _clean(_ovf(ga + EB.where(s.q_ok, (-g_exp) * _ovf(q / safe), 0.0)))     # -g * ((D / alpha) / alpha)
    dn = _rot(s.vm, grn, True)
    d_med = EB.where(s.m_ok, g_sd * EB.w(s.r), 0.0)
    chans = [d_D, d_al, dn[0], dn[1], dn[2], _clean(d_med), gds, EB(z)]
    d_allmap = EB(np.stack([x.v for x in chans]), np.stack([x.e for x in chans]))
    return d_color, d_allmap, excl


# ---------------------------------------------------------------------------------------------------------------- loss

def chain_bound(terms_abs: np.ndarray, threads: int) -> np.ndarray:
    """K * sum over each thread's grid-stride chain of |running sum| (terms in index order, thread t takes t,
    t + threads, ...): the error of the chain's fp32 additions, per thread."""
    n = terms_abs.size
    L = -(-n // threads)
    pad, real = np.zeros(L * threads), np.zeros(L * threads, bool)
    pad[:n], real[:n] = terms_abs, True
    return K * np.where(real.reshape(L, threads), np.cumsum(pad.reshape(L, threads), axis=0), 0.0).sum(0)


def loss_sums64(image, target, rend_normal, depth_normal, acc, dist, with_reg, blocks):
    """The three sums of loss_sums_kernel over V stacked views (image/rn/dn [V,3,H,W], target [V,H,W,3], acc/dist
    [V,H,W]) with a bound that follows its summation tree: a grid-stride fp32 chain per thread over ``blocks * 256``
    threads, five fp32 shuffle levels, then double (block sum, and atomics or the fixed-order finalize)."""
    img, tar = _f32(image).astype(np.float64), _f32(target).astype(np.float64)
    V, _, H, W = img.shape
    threads = int(blocks) * 256
    d = img - tar.transpose(0, 3, 1, 2)                        # [V,3,H,W]
    sq = (d * d).transpose(0, 2, 3, 1).reshape(-1, 3)          # per pixel, channels in the fma order
    sums, errs = [], []

    def reduce(term_v, term_e, steps):
        """Sum of the per-pixel terms (each with its own bound) over the kernel's tree; `steps` roundings of the
        chain per pixel, each bounded by the pixel's running sum (the terms of one pixel share a sign)."""
        n = term_v.shape[0]
        chain = steps * chain_bound(np.abs(term_v), threads)
        lane = np.zeros(-(-n // threads) * threads)
        lane[:n] = np.abs(term_v)
        lane_sum = lane.reshape(-1, threads).sum(0)                         # |thread sums| (upper bound)
        shuffles = 5 * K * lane_sum.sum()                                   # five levels within each warp
        e = float(np.sum(term_e) + chain.sum() + shuffles) + _D * (2 * int(blocks) + 64) * float(lane_sum.sum())
        return float(np.sum(term_v)), e

    # mse: three fma per pixel adding d_c^2, d_c = fl(img - tar) with its rounding (2K + K^2) d_c^2
    mse_v, mse_e = reduce(sq.sum(1), (2 * K + K * K) * sq.sum(1), 3)
    sums.append(mse_v), errs.append(mse_e)
    if with_reg:
        dv = _f32(dist).astype(np.float64).reshape(-1)
        v_, e_ = reduce(dv, np.zeros_like(dv), 1)
        sums.append(v_), errs.append(e_)
        rn = [EB(_f32(rend_normal).astype(np.float64)[:, k].reshape(-1)) for k in range(3)]
        dn = [EB(_f32(depth_normal).astype(np.float64)[:, k].reshape(-1)) for k in range(3)]
        a = _f32(acc).astype(np.float64).reshape(-1)
        one_m = 1.0 - (rn[0] * dn[0] + rn[1] * dn[1] + rn[2] * dn[2])
        t = one_m.v * a
        v_, e_ = reduce(t, one_m.e * np.abs(a), 1)
        sums.append(v_), errs.append(e_)
    else:
        sums += [0.0, 0.0]
        errs += [0.0, 0.0]
    return np.array(sums), np.array(errs)


def loss64(image, target, rend_normal, depth_normal, acc, dist, with_reg, batch_scenes, upstream, blocks):
    """One scene's share of LaRa's loss as scene_loss computes it (sums / counts in double, then fp32), and the four
    gradient maps of loss_grads_kernel for an upstream scalar.  Returns {"sums", "loss", "mse", "distortion",
    "normal"} as (value, bound) and {"image", "rend_normal", "depth_normal", "rend_dist"} as EB ([V,3,H,W] /
    [V,H,W]; None where the kernel writes nothing)."""
    s, se = loss_sums64(image, target, rend_normal, depth_normal, acc, dist, with_reg, blocks)
    img = _f32(image).astype(np.float64)
    V, _, H, W = img.shape
    npx = float(batch_scenes) * V * H * W
    mse, dst, nrm = s[0] / (3.0 * npx), s[1] / npx, s[2] / npx
    mse_e, dst_e, nrm_e = se[0] / (3.0 * npx), se[1] / npx, se[2] / npx
    loss = mse + (1000.0 * dst + 0.2 * nrm if with_reg else 0.0)
    loss_e = mse_e + (1000.0 * dst_e + 0.2 * nrm_e if with_reg else 0.0) + 4 * _D * (abs(mse) + 1000 * abs(dst) + abs(nrm))
    f = lambda v, e: (v, e + 0.5 * K * abs(v) + _D * abs(v))         # noqa: E731 (the final .float())
    vals = {"sums": (s, se), "loss": f(loss, loss_e), "mse": f(mse, mse_e), "distortion": f(dst, dst_e),
            "normal": f(nrm, nrm_e)}
    up = EB(float(np.float32(upstream)))
    tar = _f32(target).astype(np.float64).transpose(0, 3, 1, 2)
    k_mse = 2.0 * EB.w(1.0 / (3.0 * npx)) * up
    grads = {"image": k_mse * (EB(img) - EB(tar))}
    if with_reg:
        k = (-EB.w(0.2 / npx)) * up * EB(_f32(acc).astype(np.float64)[:, None])
        grads["rend_normal"] = k * EB(_f32(depth_normal).astype(np.float64))
        grads["depth_normal"] = k * EB(_f32(rend_normal).astype(np.float64))
        w = EB.w(1000.0 / npx) * up
        grads["rend_dist"] = EB(np.full((V, H, W), w.v), np.full((V, H, W), w.e))
    else:
        grads.update(rend_normal=None, depth_normal=None, rend_dist=None)
    return vals, grads


# ------------------------------------------------------------------------------------------------------------- decoder

def _sigmoid(x: EB) -> EB:
    """1 / (1 + expf(-x)) (decoder.cu's dec_sigmoid: 2-ulp expf, a correctly rounded division)."""
    return 1.0 / (1.0 + (-x).exp())


U = 2.0 ** -24                  # half an ulp, relative: one correctly rounded fp32 operation


def _rn(v, e) -> EB:
    """One correctly rounded fp32 operation: `v` its exact result on exact operands, `e` how far the exact result on the
    computed operands may lie from v.  Adds half an ulp of that result, nothing where it is exact."""
    v, e = np.asarray(v, np.float64), np.asarray(e, np.float64)
    exact = (e == 0) & (v.astype(np.float32).astype(np.float64) == v)
    return EB(v, np.where(exact, 0.0, e + U * (np.abs(v) + e)))


def _offset_vjp(g, x, half_cell) -> EB:
    """decoder.cu's offset gradient ``gc * half_cell * 2.0f * s * (1.0f - s)``, s = __fdiv_rn(1, 1 + expf(-x)),
    left to right, with half-ulp rules for its correctly rounded operations (EB's full ulp per operation makes the bound
    several times the real error where 1 - s is small): expf 2 ulp; 1 + t and the division half an ulp; 1 - s exact
    for s >= 0.5 (Sterbenz; x > 1e-3 leaves expf's error room), else half an ulp; the product by the fp32 half_cell half
    an ulp unless exact (a power of two), by 2 exact, by s and by 1 - s half an ulp each."""
    t = (-EB(x)).exp()
    a = _rn(1.0 + t.v, t.e)
    sv = 1.0 / a.v
    s = _rn(sv, sv * a.e / (a.v - a.e))
    om_v = 1.0 - s.v
    om = EB(om_v, np.where(x > 1e-3, s.e, s.e + U * (np.abs(om_v) + s.e)))
    hc32 = float(np.float32(half_cell))
    p = _rn(g * half_cell, np.abs(g) * abs(hc32 - half_cell))
    p = EB(2.0 * p.v, 2.0 * p.e)
    p = _rn(p.v * s.v, np.abs(p.v) * s.e + np.abs(s.v) * p.e + p.e * s.e)
    return _rn(p.v * om.v, np.abs(p.v) * om.e + np.abs(om.v) * p.e + p.e * om.e)


def decoder64(params, group_centers, K_, sh_dim, opacity_shift, scaling_shift, half_cell, grads=None):
    """The decoder layout of ``decoder_layout_torch``: params [B,N,K*C] -> (centers [B,N*K,3], sh [B,N*K,sh_dim/3,3],
    scaling [B,N*K,2], rotation [B,N*K,4], opacity [B,N*K,1]) as EB; with ``grads`` (the five upstream tensors,
    any None) also the gradient [B,N,K*C] as EB."""
    p = _f32(params).astype(np.float64)
    B, N = p.shape[0], p.shape[1]
    C = 10 + sh_dim
    rows = p.reshape(B, N * K_, C)
    gcn = _f32(group_centers).astype(np.float64).reshape(N, 3)
    cen = np.repeat(gcn, K_, axis=0)[None]                     # [1, N*K, 3]
    hc = EB.w(float(half_cell))
    s = _sigmoid(EB(rows[..., 0:3]))
    centers = EB(cen) + (s * 2.0 - 1.0) * hc
    out = (centers, EB(rows[..., 3:3 + sh_dim].reshape(B, N * K_, sh_dim // 3, 3)),
           EB(rows[..., 4 + sh_dim:6 + sh_dim]) + EB.w(float(scaling_shift)),
           EB(rows[..., 6 + sh_dim:10 + sh_dim]), EB(rows[..., 3 + sh_dim:4 + sh_dim]) + EB.w(float(opacity_shift)))
    if grads is None:
        return out, None
    g = [None if x is None else _f32(x).astype(np.float64) for x in grads]
    gv, ge = np.zeros((B, N * K_, C)), np.zeros((B, N * K_, C))
    if g[0] is not None:
        off = _offset_vjp(g[0].reshape(B, N * K_, 3), rows[..., 0:3], float(half_cell))
        gv[..., 0:3], ge[..., 0:3] = off.v, off.e
    if g[1] is not None:
        gv[..., 3:3 + sh_dim] = g[1].reshape(B, N * K_, sh_dim)
    if g[4] is not None:
        gv[..., 3 + sh_dim] = g[4].reshape(B, N * K_)
    if g[2] is not None:
        gv[..., 4 + sh_dim:6 + sh_dim] = g[2].reshape(B, N * K_, 2)
    if g[3] is not None:
        gv[..., 6 + sh_dim:10 + sh_dim] = g[3].reshape(B, N * K_, 4)
    return out, EB(gv.reshape(B, N, K_ * C), ge.reshape(B, N, K_ * C))
