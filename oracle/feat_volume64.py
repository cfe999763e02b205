"""Float64 statement, with a bound per element, of the coarse pass's feature-volume lifting (lara_b200/csrc/feat_volume.cu),
the forward (both layouts) and every gradient.

TEST INFRASTRUCTURE ONLY -- importable from tests/; never from lara_b200/.

Every value is an ``oracle.EB`` under ``oracle.point_feats64``'s per-operation rules: half an ulp per correctly rounded
fp32 operation (the build has no fast math, so ``sqrtf`` and ``/`` are correctly rounded), ``expf`` its 2 ulp, FMA
contraction covered because a fused operation drops one of the two roundings the bound allows.  The statement follows
the kernels' operation sequence, not torch's, and its value at float64's decisions equals
``oracle.feat_volume_torch`` run in float64:

* token features: ``d / fmaxf(sqrtf(|d|^2), 1e-12f)``, ``rsh_cart_3`` of the direction and of the moment (fp32
  constants: their rounding is in the bound), SiLU ``f / (1 + expf(-f))``;
* LayerNorm: each pass is four channel-strided sequential sums (the running-sum bound ``U sum_k |s_k|``), added in
  order, divided by C; ``rstd = 1 / sqrtf(var / C + 1e-6f)``;
* modulation: two 33-term FMA chains (32 products and the bias), order-free ``gamma(32)``; ``ln = fmaf(n, g, b)``,
  ``y = fmaf(ln, 1 + scale, shift)``;
* sample: ``point_feats64.stencil``'s tap weights (the same projection, coordinate chain and hull of an undecided
  ``floor`` as the point sampler), an FMA chain of at most 4 taps, ``gamma(m)`` for m taps; the view-embedding columns
  are exact copies;
* dL/dy: each token sums weight x dL/dout over the voxels of its four cells; the order-free bound over all m terms;
* the modulation and LayerNorm vjp per token, the two per-token channel sums as warp butterflies (5 levels) added over
  the C / 32 slices;
* the parameter gradients: per-CTA fp32 partials of at most 64 tokens (8 per warp in a chain, then 8 warps in order:
  depth 15), summed in fp64 over the CTAs, then rounded once; ``view_embed``: 64 fp32 row slices (each 8 sequential
  group sums added in order), summed in fp64, rounded once.

Bounds are formed as products of magnitudes (``|S|^T |W|`` times the order-free factor, plus the propagated bounds), per
(scene, view), so LaRa's size fits in host memory.  With zeros padding a tap's weight goes to 0 at its cell's edge, so
the sample and every gradient are continuous in (ix, iy): a ``floor`` the bound leaves undecided is held to the hull of
both sides (``hulled`` counts those voxel-views) and no element is excluded.  z = 0 exactly is decided: the voxel has no
tap, samples 0 and gets no gradient.  An infinite bound raises.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

from . import point_feats64 as P
from .oracle import EB

U = P.U
U64 = 2.0 ** -53                # double's half ulp: the fp64 sums over the CTAs and slices
TT, WARPS, VE_SLICES = 64, 8, 64
LN_EPS = 1e-6
DEPTH_CTA = TT // WARPS + WARPS - 1     # roundings a token's term passes inside one CTA: 8 chained, 7 warp adds


def _gamma(m):
    g = np.asarray(m, np.float64) * U
    return g / (1 - g)


def _ceil_div(a, b):
    return -(-a // b)


def _sum_cols(M, axis=0):
    return np.asarray(M.sum(axis)).reshape(-1)


def fma(a, b, c) -> EB:
    """fmaf: the exact product plus c, rounded once."""
    a, b, c = EB.w(a), EB.w(b), EB.w(c)
    v = a.v * b.v + c.v
    e = np.abs(a.v) * b.e + np.abs(b.v) * a.e + a.e * b.e + c.e
    return P._round(v, e, (a.e == 0) & (b.e == 0) & (c.e == 0) & P._rep(v))


def sqrt(a: EB) -> EB:
    v = np.sqrt(a.v)
    prop = v - np.sqrt(np.maximum(a.v - a.e, 0.0))
    return P._round(v, prop, (a.e == 0) & P._rep(v) & (v * v == a.v))


def seq_sum(t: EB, axis=0) -> EB:
    """fp32 sum of the terms along axis in order, from 0 (the first add is exact): with the running sums s_k,
    E <= (sum e + U sum_{k>=2} |s_k|) / (1 - (n - 1) U)."""
    n = t.v.shape[axis]
    s = np.cumsum(t.v, axis)
    run = np.abs(s).sum(axis) - np.abs(np.take(s, 0, axis))
    return EB(s.take(n - 1, axis), (t.e.sum(axis) + U * run) / (1 - (n - 1) * U))


def tree_sum(t: EB, depth, axis=0) -> EB:
    """fp32 sum of the terms along axis in a tree where no term passes more than `depth` roundings."""
    mag = (np.abs(t.v) + t.e).sum(axis)
    return EB(t.v.sum(axis), t.e.sum(axis) + _gamma(depth) * mag)


def _rsh3(x: EB, y: EB, z: EB):
    """rsh3 of feat_volume.cu, its fp32 constants as float64 constants with their rounding in the bound."""
    mul, add = P.mul, P.add
    pi = np.pi
    c1, c2, c6 = np.sqrt(3 / (4 * pi)), 0.5 * np.sqrt(15 / pi), 0.25 * np.sqrt(5 / pi)
    c8, c9, c10 = 0.25 * np.sqrt(15 / pi), 0.25 * np.sqrt(35 / (2 * pi)), 0.5 * np.sqrt(105 / pi)
    c11, c12, c14 = 0.25 * np.sqrt(21 / (2 * pi)), 0.25 * np.sqrt(7 / pi), 0.25 * np.sqrt(105 / pi)
    x2, y2, z2 = mul(x, x), mul(y, y), mul(z, z)
    xy = mul(x, y)
    one_5z2 = add(1.0, -mul(5.0, z2))
    return [EB.w(np.full(x.v.shape, 0.5 / np.sqrt(pi))), mul(-c1, y), mul(c1, z), mul(-c1, x),
            mul(c2, xy), mul(-c2, mul(y, z)), mul(c6, add(mul(3.0, z2), -1.0)), mul(-c2, mul(x, z)),
            mul(c8, add(x2, -y2)),
            mul(mul(-c9, y), add(mul(3.0, x2), -y2)), mul(mul(c10, xy), z), mul(mul(c11, y), one_5z2),
            mul(mul(c12, z), add(mul(5.0, z2), -3.0)), mul(mul(c11, x), one_5z2), mul(mul(c14, z), add(x2, -y2)),
            mul(mul(-c9, x), add(x2, -mul(3.0, y2)))]


def token_features(rays) -> EB:
    """SiLU of [rsh_cart_3(d^), rsh_cart_3(o x d^)] of rays [n, 6] (fp32 values): [n, 32]."""
    r = [EB(rays[:, k]) for k in range(6)]
    o, d = r[:3], r[3:]
    nrm = sqrt(P.sum_any_order([P.mul(d[0], d[0]), P.mul(d[1], d[1]), P.mul(d[2], d[2])]))
    inv = P.div(1.0, EB(np.maximum(nrm.v, np.float64(np.float32(1e-12))), nrm.e))
    u = [P.mul(d[k], inv) for k in range(3)]
    cross = [P.sum_any_order([P.mul(o[1], u[2]), -P.mul(o[2], u[1])]),
             P.sum_any_order([P.mul(o[2], u[0]), -P.mul(o[0], u[2])]),
             P.sum_any_order([P.mul(o[0], u[1]), -P.mul(o[1], u[0])])]
    f = _rsh3(*u) + _rsh3(*cross)
    s = [P.div(t, P.add(1.0, EB.exp(-t))) for t in f]
    return EB(np.stack([t.v for t in s], 1), np.stack([t.e for t in s], 1))


def _cols(a: EB, sl):
    return EB(a.v[:, sl], a.e[:, sl])


class _Tokens:
    """The token forward of one (scene, view): x [C, n] (fp32 values), rays [n, 6] -> S, mean, rstd, n, ln, 1 + scale,
    y, each [n, ...]."""

    def __init__(self, x, rays, ln_w, ln_b, mlp_w, mlp_b):
        C = x.shape[0]
        self.S = token_features(rays)
        xt = x.T                                                          # [n, C]
        parts = xt.reshape(xt.shape[0], C // 4, 4)                        # channel 4 q + p: part p, step q
        s = seq_sum(EB(parts), axis=1)                                    # [n, 4]
        tot = P.add(P.add(P.add(_cols(s, 0), _cols(s, 1)), _cols(s, 2)), _cols(s, 3))
        self.mean = P.div(tot, float(C))
        m = EB(self.mean.v[:, None], self.mean.e[:, None])
        d = P.add(EB(xt), -m)                                             # [n, C]
        sq = EB((d.v * d.v).reshape(parts.shape), (2 * np.abs(d.v) * d.e + d.e * d.e).reshape(parts.shape))
        s = seq_sum(sq, axis=1)
        tot = P.add(P.add(P.add(_cols(s, 0), _cols(s, 1)), _cols(s, 2)), _cols(s, 3))
        self.rstd = P.div(1.0, sqrt(P.add(P.div(tot, float(C)), LN_EPS)))
        r = EB(self.rstd.v[:, None], self.rstd.e[:, None])
        self.n = P.mul(d, r)
        self.ln = fma(self.n, ln_w[None], ln_b[None])
        Sa = np.abs(self.S.v) + self.S.e
        Wa = np.abs(mlp_w)
        lin = self.S.v @ mlp_w.T + mlp_b                                  # [n, 2C]: 32 products and the bias
        lin_e = self.S.e @ Wa.T + _gamma(32) * (Sa @ Wa.T + np.abs(mlp_b))
        self.sh, sc = EB(lin[:, :C], lin_e[:, :C]), EB(lin[:, C:], lin_e[:, C:])
        self.one_sc = P.add(1.0, sc)
        self.y = fma(self.ln, self.one_sc, self.sh)


def cond_rows(B, V, R, n_group):
    """Row of each voxel of each (scene, view) in the condition layout [B g^3, V bs^3, C+E]: [B, V, R^3]."""
    bs = R // n_group
    g = np.arange(R ** 3)
    i, j, k = g // (R * R), (g // R) % R, g % R
    G = ((i // bs) * n_group + j // bs) * n_group + k // bs
    lo = ((i % bs) * bs + j % bs) * bs + k % bs
    b, v = np.arange(B)[:, None, None], np.arange(V)[None, :, None]
    return (b * n_group ** 3 + G) * (V * bs ** 3) + v * bs ** 3 + lo


def canonical(t, B, V, C, R, n_group):
    """An output or upstream of either layout as [B, V, R^3, C] and (condition layout) its view-embedding columns
    [B, V, R^3, E] (None in the drop-in layout)."""
    a = t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)
    if n_group == 0:
        return a.reshape(B, V, C, R ** 3).transpose(0, 1, 3, 2), None
    rows = a.reshape(-1, a.shape[-1])[cond_rows(B, V, R, n_group)]
    return rows[..., :C], rows[..., C:]


def _weights_matrix(st, h, w, R3):
    """Sparse [R3, h w] matrices of the stencil's weight values and of their spread + rounding, and per voxel the
    number of taps some side uses."""
    t = st["touched"]
    s_, vox = np.nonzero(t)
    pix = (st["Y"][s_, vox] * w + st["X"][s_, vox]).astype(np.int64)
    shape = (R3, h * w)
    Wv = sp.csr_matrix((st["v"][s_, vox], (vox, pix)), shape)
    Wd = sp.csr_matrix((st["d"][s_, vox] + st["r"][s_, vox], (vox, pix)), shape)
    Wn = sp.csr_matrix((np.ones(vox.size), (vox, pix)), shape)
    return Wv, Wd, Wn, t.sum(0)


def _final(v, prop, mag, nparts):
    """A per-CTA (or per-slice) fp32 partial sum's value and bound, summed in fp64 over nparts, rounded once to fp32."""
    e = prop + (nparts - 1) * U64 * mag / (1 - nparts * U64)
    return P._round(v, e, np.zeros(np.shape(v), bool))


def feat_volume64(img_feats, rays, w2cs, ixts, image_hw, grid, params, grads=()):
    """img_feats [B V,C,h,w], rays [B,V,h,w,6], w2cs [B,V,4,4], ixts [B,V,3,3], image_hw = (H_img, W_img), grid
    [R,R,R,3], params = (norm.weight, norm.bias, mlp.1.weight, mlp.1.bias); grads: upstream gradients, each a pair
    (G [B,V,R^3,C], GE [B,V,R^3,E] or None) in ``canonical`` form.

    Returns ``out`` EB [B,V,R^3,C] (either layout's sample, canonical), and for each upstream a dict of ``g_img_feats``
    [B V,C,h,w], ``g_norm_w``, ``g_norm_b`` [C], ``g_mlp_w`` [2C,32], ``g_mlp_b`` [2C] and (GE given, E > 0)
    ``g_view_embed`` [V,E]; ``hulled`` [B,V,R^3], the voxel-views whose floor the bound leaves undecided; ``max_terms``,
    the most (voxel, tap) terms one token's dL/dy sums."""
    f64 = P._f64
    x = f64(img_feats)
    BV, C, h, w = x.shape
    ry, E2, K3 = f64(rays), f64(w2cs), f64(ixts)
    B, V = ry.shape[:2]
    pts = f64(grid).reshape(-1, 3)
    R3 = pts.shape[0]
    ln_w, ln_b, mlp_w, mlp_b = (f64(p) for p in params)
    H_img, W_img = (int(s) for s in image_hw)
    G = [(np.asarray(g, np.float32).astype(np.float64), None if ge is None else np.asarray(ge, np.float32).astype(np.float64))
         for g, ge in grads]
    ov, oe = np.zeros((B, V, R3, C)), np.zeros((B, V, R3, C))
    hulled = np.zeros((B, V, R3), bool)
    max_terms = 0
    acc = [dict(gx=np.zeros((BV, C, h * w)), gxe=np.zeros((BV, C, h * w)),
                **{k: [0.0, 0.0, 0.0] for k in ("w_sh", "w_sc", "b_sh", "b_sc", "nw", "nb")}) for _ in G]

    def add_fma_sum(slot, a: EB, b: EB):
        """sum over the tokens of the exact products a^T b (FMA accumulators): value, propagated, magnitude."""
        Aa, Ba = np.abs(a.v), np.abs(b.v)
        slot[0] = slot[0] + a.v.T @ b.v
        slot[1] = slot[1] + Aa.T @ b.e + a.e.T @ Ba + a.e.T @ b.e
        slot[2] = slot[2] + (Aa + a.e).T @ (Ba + b.e)

    def add_sum(slot, t: EB):
        slot[0] = slot[0] + t.v.sum(0)
        slot[1] = slot[1] + t.e.sum(0)
        slot[2] = slot[2] + (np.abs(t.v) + t.e).sum(0)

    for b in range(B):
        for v in range(V):
            bv = b * V + v
            tok = _Tokens(x[bv].reshape(C, h * w), ry[b, v].reshape(h * w, 6), ln_w, ln_b, mlp_w, mlp_b)
            vw = P._View(pts, E2[b, v], K3[b, v], w, h, W_img, H_img)
            if vw.inf.any():
                raise AssertionError(f"feat_volume64: {int(vw.inf.sum())} voxels of (scene {b}, view {v}) with an "
                                     "infinite bound")
            und = vw.ax["und"] | vw.ay["und"]
            hulled[b, v] = und
            Wv, Wd, Wn, m = _weights_matrix(P.stencil(vw, w, h, und), h, w, R3)
            Wa = abs(Wv) + Wd
            y = tok.y
            ya = np.abs(y.v)
            ov[b, v] = Wv @ y.v
            oe[b, v] = Wd @ ya + Wa @ y.e + _gamma(m)[:, None] * (Wa @ (ya + y.e))
            mt = _sum_cols(Wn)
            max_terms = max(max_terms, int(mt.max()) if mt.size else 0)
            for (g, _), a in zip(G, acc):
                gb = g[b, v]
                gab = np.abs(gb)
                dy = EB(Wv.T @ gb, Wd.T @ gab + _gamma(mt)[:, None] * (Wa.T @ gab))           # [hw, C]
                dsc, dln = P.mul(dy, tok.ln), P.mul(dy, tok.one_sc)
                add_fma_sum(a["w_sh"], dy, tok.S)
                add_fma_sum(a["w_sc"], dsc, tok.S)
                add_sum(a["b_sh"], dy)
                add_sum(a["b_sc"], dsc)
                nn = tok.n
                a["nw"][0] = a["nw"][0] + (dln.v * nn.v).sum(0)
                a["nw"][1] = a["nw"][1] + (np.abs(dln.v) * nn.e + dln.e * np.abs(nn.v) + dln.e * nn.e).sum(0)
                a["nw"][2] = a["nw"][2] + ((np.abs(dln.v) + dln.e) * (np.abs(nn.v) + nn.e)).sum(0)
                add_sum(a["nb"], dln)
                # LayerNorm vjp: dx = rstd (dn - mean(dn) - n mean(dn n))
                dn = P.mul(dln, EB(ln_w[None]))
                depth = 5 + C // 32 - 1
                s1 = tree_sum(dn, depth, axis=1)
                s2 = tree_sum(P.mul(dn, nn), depth, axis=1)
                m1, m2 = P.div(s1, float(C)), P.div(s2, float(C))
                col = lambda q: EB(q.v[:, None], q.e[:, None])              # noqa: E731
                gx = P.mul(col(tok.rstd), P.add(P.add(dn, -col(m1)), -P.mul(nn, col(m2))))
                a["gx"][bv], a["gxe"][bv] = gx.v.T, gx.e.T
    ntiles = _ceil_div(h * w, TT)
    nparts = B * V * ntiles
    res = []
    for (g, ge), a in zip(G, acc):
        d = {"g_img_feats": EB(a["gx"].reshape(BV, C, h, w), a["gxe"].reshape(BV, C, h, w))}

        def part(k):
            val, prop, mag = a[k]
            return _final(val, prop + _gamma(DEPTH_CTA) * mag, mag * (1 + _gamma(DEPTH_CTA)), nparts)

        d["g_norm_w"], d["g_norm_b"] = part("nw"), part("nb")
        ws, wc, bs_, bc = part("w_sh"), part("w_sc"), part("b_sh"), part("b_sc")
        d["g_mlp_w"] = EB(np.concatenate([ws.v, wc.v]), np.concatenate([ws.e, wc.e]))
        d["g_mlp_b"] = EB(np.concatenate([bs_.v, bc.v]), np.concatenate([bs_.e, bc.e]))
        if ge is not None and ge.shape[-1] > 0:
            n = B * R3
            rows = _ceil_div(_ceil_div(n, VE_SLICES), WARPS)   # rows one group of one slice sums, at most
            gv = ge.transpose(1, 0, 2, 3).reshape(V, n, -1)    # [V, B R^3, E]
            mag = np.abs(gv).sum(1)
            val = gv.sum(1)
            d["g_view_embed"] = _final(val, _gamma(rows - 1 + WARPS - 1) * mag, mag * (1 + _gamma(rows + WARPS)),
                                       VE_SLICES)
        res.append(d)
    return {"out": EB(ov, oe), "grads": res, "hulled": hulled, "max_terms": max_terms}
