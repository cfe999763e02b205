"""Float64 statement, with a bound per element, of the VolTransformer's fused kernels: the group cross-attention
(lara_b200/csrc/vol_transformer.cu, ``ga_fwd_kernel`` / ``ga_bwd_kernel``) and the residual add + LayerNorm
(lara_b200/csrc/layer_norm.cuh, ``ln_fwd_kernel`` / ``ln_bwd_kernel``, behind both ``srf_add_layernorm`` and
``srf_vit_layernorm``), forward and every gradient.

TEST INFRASTRUCTURE ONLY -- importable from tests/; never from lara_b200/.

Every value is an ``oracle.EB`` under ``oracle.point_feats64``'s and ``oracle.feat_volume64``'s per-operation rules:
half an ulp per correctly rounded fp32 operation (no fast math: ``/`` and ``sqrtf`` are correctly rounded), ``expf``
its 2 ulp, an FMA chain as a sum of exact products whose first term is rounded too.  A contracted multiply-add drops
one of the two roundings the bound allows, so the bound holds with or without contraction.  The statement follows the
kernels' operation order, not torch's; its value equals ``oracle.vol_transformer_torch.group_attention_cl`` and
``F.layer_norm`` run in float64.

Group attention, per (query, head) thread, D = C / H:

* scores: a D-term FMA chain times the kernel's ``scale = 1 / sqrtf(D)``, whose rounding against ``D ** -0.5`` is in
  the bound (none for D = 16); ``m`` the running ``fmaxf`` of the rounded scores.  The exp pass may contract
  ``dot * scale - m`` into one FMA, so the argmax key's weight is not assumed to be exactly 1.
* The maximum cancels between numerator and denominator: its error ``delta`` (at most the largest score bound) enters
  only through the rounding of ``s - m``.  ``e_j = expf(s_j - m)`` carries expf's 2 ulp plus an absolute floor of two
  subnormal ulps, and every rounding here an underflow term of half a subnormal ulp (``TINY``), so weights and
  products in the subnormal or zero range are held to an absolute bound, not a relative one.
* forward: ``sum`` and the ``acc`` FMA chains over the keys (order-free ``gamma(S)``), ``o = acc * fl(1 / sum)``.
* backward: ``pd`` an FMA chain over the keys, ``di = pd * inv``, ``p_j = expf(...) * inv`` (rounded once more than the
  forward's weight), ``ds_j = p_j (dot(dO, v_j) - di)`` with the absolute bounds of both operands (the cancellation
  stays in the bound), ``dq = scale * sum_j ds_j k_j``; ``dv[G, j]`` and ``dk[G, j] / scale`` the sequential sums, in
  unfold order over the bs^3 queries, of the products ``p dO`` and ``ds q`` each rounded into shared memory: a term
  passes at most bs^3 roundings, so the order-free ``gamma(bs^3)`` covers that order (the sums are formed as matmuls,
  which keeps g = 8's 64 queries x 32 keys fast).

LayerNorm, a warp per row, lane l holding channels l + 32 j:

* ``y = a + b`` one rounding (none without b); the lane's ``nj = C / 32`` values summed in order, a 5-level xor
  butterfly, ``/ C``; the centred variance as an FMA chain, the butterfly, ``/ C + eps`` (eps as the fp32 the kernel
  receives: its rounding is in the bound), ``1 / sqrtf``; ``n = fmaf((y - mean) * rstd, gamma, beta)``.
* backward from y (the forward's y with its bound): the same statistics, ``gg = g * gamma`` and ``yh = (y - mean) *
  rstd`` each rounded, the lane chains ``s1`` (sum) and ``s2`` (FMA) with their butterflies, ``d = rstd (gg - m1 -
  yh m2)``, ``da = dy + d``.  dgamma / dbeta: each warp chains its rows r0 + w, r0 + w + 8, ... of a 64-row CTA, the
  8 warps added in warp order (depth 15), the CTAs' partials added in fp64 and rounded once.

No element needs a hull: the attention has no discrete decision that changes its result and the LayerNorm no branch.
An infinite bound raises.  Groups and rows are processed in chunks so that LaRa's size fits in host memory.
"""
from __future__ import annotations

import numpy as np

from . import feat_volume64 as F
from . import point_feats64 as P
from .oracle import EB

U = P.U
TINY = 2.0 ** -150              # half a subnormal ulp: the absolute part of one fp32 rounding
EXP_FLOOR = 2.0 ** -148         # expf's 2 ulp where its result is subnormal or flushed to 0
LN_ROWS, LN_WARPS = 64, 8       # rows per CTA of ln_bwd_kernel, warps per CTA
LN_DEPTH = LN_ROWS // LN_WARPS + LN_WARPS - 1
CHUNK = 1 << 22                 # elements of the largest intermediate array per chunk


def _tiny(a: EB, n=1) -> EB:
    return EB(a.v, a.e + n * TINY)


def _raise_inf(name, e):
    if not np.isfinite(e).all():
        raise AssertionError(f"vol_transformer64: {int((~np.isfinite(e)).sum())} elements of {name} with an infinite "
                             "bound")


def kernel_scale(D) -> EB:
    """``1.0f / sqrtf((float)D)`` against ``D ** -0.5``: two correctly rounded operations."""
    return P.div(1.0, F.sqrt(EB(np.float64(D))))


def _fma_sum(a, b, ea, eb_, n):
    """An n-term FMA chain of the exact products a b (matmul operands, their bounds ea, eb_), in any order: the
    products' propagated bound plus gamma(n) of the magnitudes."""
    Aa, Ba = np.abs(a) + ea, np.abs(b) + eb_
    e = np.abs(a) @ eb_ + ea @ np.abs(b) + ea @ eb_
    return EB(a @ b, e + F._gamma(n) * (Aa @ Ba) + n * TINY)


# ---------------------------------------------------------------------------------------------------- group attention

def _heads(x, G, n, H, D):
    """[G, n, C] -> [G, H, n, D]."""
    return x.reshape(G, n, H, D).transpose(0, 2, 1, 3)


def _unheads(x: EB):
    G, H, n, D = x.v.shape
    f = lambda a: a.transpose(0, 2, 1, 3).reshape(G, n, H * D)          # noqa: E731
    return f(x.v), f(x.e)


def _to_groups(x, g):
    """[B,R,R,R,C] -> [B g^3, bs^3, C] in LaRa's unfold order (the kernels' ga_voxel)."""
    B, R, _, _, C = x.shape
    bs = R // g
    return x.reshape(B, g, bs, g, bs, g, bs, C).transpose(0, 1, 3, 5, 2, 4, 6, 7).reshape(B * g ** 3, bs ** 3, C)


def _from_groups(x, B, R, g):
    bs, C = R // g, x.shape[-1]
    return x.reshape(B, g, g, g, bs, bs, bs, C).transpose(0, 1, 4, 2, 5, 3, 6, 7).reshape(B, R, R, R, C)


def _attn_chunk(q, k, v, go, sc: EB, D):
    """One chunk of groups: q, go [Gc,H,L,D], k, v [Gc,H,S,D] (fp32 values as float64) -> o, dq [Gc,H,L,D],
    dk, dv [Gc,H,S,D] as EB (dq ... None without go)."""
    L, S = q.shape[2], k.shape[2]
    z = np.zeros_like
    kt = k.transpose(0, 1, 3, 2)
    dot = _fma_sum(q, kt, z(q), z(kt), D)                                     # [Gc,H,L,S]
    s = _tiny(P.mul(dot, sc))
    delta = s.e.max(-1, keepdims=True)                                        # |fl(m) - m|
    m = s.v.max(-1, keepdims=True)
    t = s.v - m
    et = s.e + U * (np.abs(t) + s.e + delta) + TINY
    w = EB.exp(EB(t, et))
    w = EB(w.v, w.e + EXP_FLOOR)                                              # e_j = expf(s_j - m)
    tot = _tiny(F.tree_sum(w, S - 1, axis=-1), S)                            # sum, from 0 in key order
    inv = _tiny(P.div(1.0, tot))                                              # [Gc,H,L]
    acc = _fma_sum(w.v, v, w.e, z(v), S)
    col = lambda a: EB(a.v[..., None], a.e[..., None])                        # noqa: E731
    o = _tiny(P.mul(acc, col(inv)))
    if go is None:
        return o, None, None, None
    vt = v.transpose(0, 1, 3, 2)
    wd = _fma_sum(go, vt, z(go), z(vt), D)                                    # dot(dO, v_j) [Gc,H,L,S]
    pd = _fma_sum(w.v[..., None, :], wd.v[..., :, None], w.e[..., None, :], wd.e[..., :, None], S)
    pd = EB(pd.v[..., 0, 0], pd.e[..., 0, 0])
    di = _tiny(P.mul(pd, inv))
    p = _tiny(P.mul(w, col(inv)))
    ds = _tiny(P.mul(p, _tiny(P.add(wd, -col(di)))))
    gq = _tiny(P.mul(_fma_sum(ds.v, k, ds.e, z(k), S), sc))
    # the staged products p dO and ds q, each rounded once, then L - 1 sequential adds over the queries
    tr = lambda a: a.swapaxes(-1, -2)                                         # noqa: E731
    gv = _tiny(_fma_sum(tr(p.v), go, tr(p.e), z(go), L), L)
    gk = _tiny(P.mul(_tiny(_fma_sum(tr(ds.v), q, tr(ds.e), z(q), L), L), sc))
    return o, gq, gk, gv


def group_attention64(q, k, v, g, H, go=None):
    """q [B,R,R,R,C], k, v [B g^3, S, C], go (dL/do, like q, or None) -> {"o", and with go "dq", "dk", "dv"} as EB in
    the layouts of q and k."""
    f64 = P._f64
    q, k, v = f64(q), f64(k), f64(v)
    B, R, C = q.shape[0], q.shape[1], q.shape[-1]
    G, S = k.shape[0], k.shape[1]
    D = C // H
    L = (R // g) ** 3
    sc = kernel_scale(D)
    qg = _to_groups(q, g)
    gog = None if go is None else _to_groups(f64(go), g)
    out = {n: (np.zeros(qg.shape), np.zeros(qg.shape)) for n in ("o", "dq")}
    out.update({n: (np.zeros(k.shape), np.zeros(k.shape)) for n in ("dk", "dv")})
    step = max(1, CHUNK // (H * L * max(S, D)))
    for g0 in range(0, G, step):
        sl = slice(g0, min(G, g0 + step))
        n = sl.stop - sl.start
        res = _attn_chunk(_heads(qg[sl], n, L, H, D), _heads(k[sl], n, S, H, D), _heads(v[sl], n, S, H, D),
                          None if go is None else _heads(gog[sl], n, L, H, D), sc, D)
        for name, r in zip(("o", "dq", "dk", "dv"), res):
            if r is not None:
                out[name][0][sl], out[name][1][sl] = _unheads(r)
    res = {"o": EB(*(_from_groups(a, B, R, g) for a in out["o"]))}
    if go is not None:
        res["dq"] = EB(*(_from_groups(a, B, R, g) for a in out["dq"]))
        res["dk"], res["dv"] = EB(*out["dk"]), EB(*out["dv"])
    for name, r in res.items():
        _raise_inf(name, r.e)
    return res


# --------------------------------------------------------------------------------------------------------- LayerNorm

def _lanes(x: EB, nj):
    """[rows, C] -> [rows, nj, 32]: lane l's values l + 32 j along axis 1."""
    return EB(x.v.reshape(-1, nj, 32), x.e.reshape(-1, nj, 32))


def _row(x: EB, C):
    """A lane sum [rows, 32] -> its butterfly total / C, [rows, 1]."""
    t = F.tree_sum(x, 5, axis=1)
    r = P.div(EB(t.v[:, None], t.e[:, None]), float(C))
    return r


def _fma_chain(t: EB, axis=1) -> EB:
    """An FMA chain from 0 over the exact products t along axis: seq_sum with the first product's rounding."""
    first = np.zeros(t.v.shape[axis], bool)
    first[0] = True
    shape = [1] * t.v.ndim
    shape[axis] = -1
    f = first.reshape(shape)
    return F.seq_sum(EB(t.v, t.e + np.where(f, U * np.abs(t.v), 0.0)), axis)


def _stats(y: EB, C, eps):
    """ln_stats: mean, rstd [rows, 1] and d = y - mean [rows, C]."""
    nj = C // 32
    mean = _row(F.seq_sum(_lanes(y, nj), axis=1), C)
    d = P.add(y, -mean)
    sq = EB(d.v * d.v, 2 * np.abs(d.v) * d.e + d.e * d.e)
    var = _row(_fma_chain(_lanes(sq, nj)), C)
    rstd = P.div(1.0, F.sqrt(P.add(var, EB.w(np.float64(eps)))))
    return mean, rstd, d


def layer_norm64(a, b, gamma, beta, eps, gn=None, gy=None):
    """a, b (or None) [rows, C], gamma, beta [C]; gn = dL/dn (or None for no backward), gy = dL/dy (or None) ->
    {"y", "n"} and with gn {"da", "dgamma", "dbeta"}, as EB.  eps the module's (float64) value."""
    f64 = P._f64
    a = f64(a)
    rows, C = a.shape
    b = None if b is None else f64(b)
    gam, bet = f64(gamma), f64(beta)
    gn = None if gn is None else f64(gn)
    gy = None if gy is None else f64(gy)
    nj = C // 32
    keys = ("y", "n") + (() if gn is None else ("da",))
    out = {k: (np.zeros((rows, C)), np.zeros((rows, C))) for k in keys}
    # dgamma / dbeta: value, propagated bound, magnitude, summed over the rows
    acc = {k: [np.zeros(C), np.zeros(C), np.zeros(C)] for k in ("dgamma", "dbeta")}
    step = max(LN_ROWS, CHUNK // C // LN_ROWS * LN_ROWS)
    G, Bt = EB(gam[None]), EB(bet[None])
    for r0 in range(0, rows, step):
        sl = slice(r0, min(rows, r0 + step))
        y = EB(a[sl]) if b is None else P.add(EB(a[sl]), EB(b[sl]))
        mean, rstd, d = _stats(y, C, eps)
        yh = P.mul(d, rstd)
        n = F.fma(yh, G, Bt)
        out["y"][0][sl], out["y"][1][sl] = y.v, y.e
        out["n"][0][sl], out["n"][1][sl] = n.v, n.e
        if gn is None:
            continue
        g = gn[sl]
        gg = P.mul(EB(g), G)
        s1 = F.seq_sum(_lanes(gg, nj), axis=1)
        prod = EB(gg.v * yh.v, np.abs(gg.v) * yh.e + gg.e * np.abs(yh.v) + gg.e * yh.e)
        s2 = _fma_chain(_lanes(prod, nj))
        m1, m2 = _row(s1, C), _row(s2, C)
        dd = P.mul(rstd, P.add(P.add(gg, -m1), -P.mul(yh, m2)))
        da = dd if gy is None else P.add(EB(gy[sl]), dd)
        out["da"][0][sl], out["da"][1][sl] = da.v, da.e
        ga = np.abs(g)
        for k, val, prop, mag in (("dgamma", g * yh.v, ga * yh.e, ga * (np.abs(yh.v) + yh.e)),
                                  ("dbeta", g, np.zeros_like(g), ga)):
            acc[k][0] += val.sum(0)
            acc[k][1] += prop.sum(0)
            acc[k][2] += mag.sum(0)
    res = {k: EB(*out[k]) for k in keys}
    if gn is not None:
        nparts = -(-rows // LN_ROWS)
        for k, (val, prop, mag) in acc.items():
            res[k] = F._final(val, prop + F._gamma(LN_DEPTH) * mag, mag * (1 + F._gamma(LN_DEPTH)), nparts)
    for name, r in res.items():
        _raise_inf(name, r.e)
    return res
