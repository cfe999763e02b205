"""The VolTransformer's fused kernels element by element against float64: the group cross-attention
(csrc/vol_transformer.cu) and the residual add + LayerNorm (csrc/layer_norm.cuh) through both of its entries,
``srf_add_layernorm`` (the VolTransformer's blocks) and ``srf_vit_layernorm`` (the DINO encoder's blocks).

``oracle.vol_transformer64`` restates the kernels' operation order in float64 with a bound per element on what their
fp32 evaluation may differ by (its docstring derives the rules).  So the dv / dk of a key whose softmax weight is
2^-100, an output of a query whose every score is below -100, and a LayerNorm row a thousand away from 0 or with a
variance near eps are each held to their own bound, not to a fraction of the tensor's largest element.

CPU part: the statement equals ``group_attention_cl`` and ``F.layer_norm`` (and their autograd gradients) run in
float64; the fp32 torch restatements and an fp32 NumPy emulation of the kernels' exact operation order (FMA as one
float64 operation rounded to fp32) lie within the bound at every element.  GPU part: the forward and every gradient
at LaRa's sizes and at the head counts, block sizes, key counts, score ranges, channel counts, row counts and row
shapes the kernels treat differently; exactly constant rows normalise to beta bit for bit, and zero rows give exact
zero dgamma / dbeta.
"""
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import vol_transformer64 as VT
from test_chain_per_element import _pin64, _tightness
from test_feat_volume_per_element import _butterfly, _fma
from test_point_feats_per_element import _check

f32, f64 = np.float32, np.float64
ATTN_OUT = ("o", "dq", "dk", "dv")
LN_OUT = ("y", "n", "da", "dgamma", "dbeta")


# ------------------------------------------------------------------------------------------------------------- inputs

def attn_inputs(B, R, g, S, C, H, scores, seed):
    """q [B,R,R,R,C], k, v [B g^3, S, C], dL/do (fp32, CPU).  scores: "randn" (unit inputs); "top100" (q scaled so
    that the largest score is 100); "below100" (every score of every query below -100, spread ~10 within a query);
    "spread" (each query's scores spread over ~85: weights down to the subnormal range)."""
    from oracle.vol_transformer_torch import from_groups, to_groups
    gen = torch.Generator().manual_seed(seed)
    D, G, L = C // H, B * g ** 3, (R // g) ** 3
    q = torch.randn((B, R, R, R, C), generator=gen, dtype=torch.float64)
    k = torch.randn((G, S, C), generator=gen, dtype=torch.float64)
    v = torch.randn((G, S, C), generator=gen)
    up = torch.randn((B, R, R, R, C), generator=gen)
    if scores == "top100":
        s = to_groups(q, g).view(G, L, H, D).transpose(1, 2) @ k.view(G, S, H, D).permute(0, 2, 3, 1) / D ** 0.5
        q = q * (100.0 / float(s.max()))
    elif scores in ("below100", "spread"):
        # a unit direction u per (group, head): q = A u + noise, k_j = c_j u + noise, so s_lj ~ A c_j / sqrt(D)
        u = torch.randn((G, 1, H, D), generator=gen, dtype=torch.float64)
        u = u / u.norm(dim=-1, keepdim=True)
        if scores == "below100":
            A, c, nq, nk = 30.0, torch.full((G, S, 1, 1), -30.0, dtype=torch.float64), 1.0, 1.0
        else:
            A, nq, nk = 10.0, 0.3, 0.3
            top = 4.0 * D ** 0.5 / A         # scores from ~+4 down to ~-81 within each query, keys in random order
            lin = torch.linspace(top, top - 85.0 * D ** 0.5 / A, S, dtype=torch.float64) if S > 1 else \
                torch.tensor([top], dtype=torch.float64)
            c = torch.stack([lin[torch.randperm(S, generator=gen)] for _ in range(G)]).view(G, S, 1, 1)
        qg = A * u + nq * to_groups(q, g).view(G, L, H, D)
        q = from_groups(qg.reshape(G, L, C), B, R, g)
        k = (c * u + nk * k.view(G, S, H, D)).reshape(G, S, C)
    return q.float().contiguous(), k.float().contiguous(), v, up


def scores64(q, k, g, H):
    from oracle.vol_transformer_torch import to_groups
    G, S, C = k.shape
    D = C // H
    qg = to_groups(q.double(), g)
    return qg.view(G, -1, H, D).transpose(1, 2) @ k.double().view(G, S, H, D).permute(0, 2, 3, 1) / D ** 0.5


def ln_inputs(rows, C, eps, has_b, seed):
    """a, b (or None), dL/dn, dL/dy, gamma, beta (fp32, CPU), and the rows that are exactly constant.  Rows by
    index mod 8: 0 offset by ~1e3 with unit spread, 1 one massive channel (~300) among N(0, 1), 2 exactly constant,
    3 near-constant (variance ~ eps), the others ``randn * 2 + 0.5`` (+ randn)."""
    gen = torch.Generator().manual_seed(seed)
    a = torch.randn((rows, C), generator=gen) * 2 + 0.5
    b = torch.randn((rows, C), generator=gen) if has_b else None
    r = torch.arange(rows) % 8
    n0 = torch.randn((rows, C), generator=gen)
    off, big, const, near = (r == 0), (r == 1), (r == 2), (r == 3)
    a[off] = 1000.0 + 0.7 * n0[off]
    a[big] = n0[big]
    a[big, 37 % C] = 300.0 + n0[big, 0]
    lvl = (torch.arange(rows, dtype=torch.float32) % 13 - 6) * 0.75    # exact sums with b's constant
    a[const] = lvl[const, None]
    a[near] = -0.3 + eps ** 0.5 * n0[near]
    if b is not None:
        b[off] = 0.7 * torch.randn((int(off.sum()), C), generator=gen)
        b[big] = 0.0
        b[const] = 2.5
        b[near] = 0.0
    gn, gy = torch.randn((rows, C), generator=gen), torch.randn((rows, C), generator=gen)
    w, bb = 1 + 0.2 * torch.randn(C, generator=gen), 0.1 * torch.randn(C, generator=gen)
    return a, b, gn, gy, w, bb, const.numpy()


# --------------------------------------------------------------------------------------------------------- checking

def _np(t):
    return t.detach().cpu().numpy().astype(f64)


def check_all(res, st, names, ctx):
    """Every element of every output within its bound; prints the worst err/bound and the tightness."""
    worst = {n: _check(res[n], st[n], f"{ctx} {n}") for n in names if n in st}
    print(f"\n  {ctx}: worst err/bound " + ", ".join(f"{n} {v:.3g}" for n, v in worst.items()) +
          f"; statement {st['seconds']:.1f} s")
    for n in worst:
        _tightness(n, st[n])
    return worst


def attn_statement(q, k, v, up, g, H):
    t0 = time.perf_counter()
    st = VT.group_attention64(q, k, v, g, H, up)
    st["seconds"] = time.perf_counter() - t0
    return st


def ln_statement(a, b, gn, gy, w, bb, eps):
    t0 = time.perf_counter()
    st = VT.layer_norm64(a, b, w, bb, eps, gn, gy)
    st["seconds"] = time.perf_counter() - t0
    return st


def torch_attention(q, k, v, up, g, H, dtype):
    from oracle.vol_transformer_torch import group_attention_cl
    ins = [t.to(dtype).clone().requires_grad_(True) for t in (q, k, v)]
    o = group_attention_cl(*ins, g, H)
    o.backward(up.to(dtype))
    return {"o": _np(o), "dq": _np(ins[0].grad), "dk": _np(ins[1].grad), "dv": _np(ins[2].grad)}


def torch_layer_norm(a, b, gn, gy, w, bb, eps, dtype):
    ins = [t.to(dtype).clone().requires_grad_(True) if t is not None else None for t in (a, b, w, bb)]
    y = ins[0] + ins[1] if b is not None else ins[0]
    n = F.layer_norm(y, (a.shape[1],), ins[2], ins[3], eps)
    has_dy = gy is not None and b is not None
    torch.autograd.backward([n] + ([y] if has_dy else []), [gn.to(dtype)] + ([gy.to(dtype)] if has_dy else []))
    return {"y": _np(y), "n": _np(n), "da": _np(ins[0].grad), "dgamma": _np(ins[2].grad), "dbeta": _np(ins[3].grad)}


# ------------------------------------------------------------------------------------------- fp32 emulation (NumPy)

def emulate_attention(q, k, v, up, g, H):
    """ga_fwd_kernel and ga_bwd_kernel's operation order in fp32: per (query, head) the D-term FMA dots, the running
    fmaxf, expf, the key-order sum and FMA accumulators, o = acc * (1 / sum); the backward's staged products summed
    over the queries in unfold order."""
    qg = VT._to_groups(q.numpy(), g)
    G, L, C = qg.shape
    S, D = k.shape[1], C // H
    hq = lambda x, n: x.reshape(G, n, H, D).transpose(0, 2, 1, 3)          # noqa: E731
    Q, GO = hq(qg, L), hq(VT._to_groups(up.numpy(), g), L)
    K, V = hq(k.numpy(), S), hq(v.numpy(), S)
    sc = f32(1) / np.sqrt(f32(D))

    def dot(x, y):
        s = np.zeros(x.shape[:3], f32)
        for i in range(D):
            s = _fma(x[..., i], y[:, :, None, i], s)
        return s
    dots = [dot(Q, K[:, :, j]) for j in range(S)]
    m = np.full(Q.shape[:3], -np.inf, f32)
    for j in range(S):
        m = np.maximum(m, dots[j] * sc)
    with np.errstate(under="ignore"):
        e = [np.exp(dots[j] * sc - m) for j in range(S)]
    tot, acc = np.zeros(Q.shape[:3], f32), np.zeros(Q.shape, f32)
    for j in range(S):
        tot = tot + e[j]
        acc = _fma(e[j][..., None], V[:, :, None, j], acc)
    inv = f32(1) / tot
    o = acc * inv[..., None]
    wd = [dot(GO, V[:, :, j]) for j in range(S)]
    pd = np.zeros(Q.shape[:3], f32)
    for j in range(S):
        pd = _fma(e[j], wd[j], pd)
    di = pd * inv
    gq = np.zeros(Q.shape, f32)
    gk, gv = np.zeros(K.shape, f32), np.zeros(K.shape, f32)
    with np.errstate(under="ignore"):
        for j in range(S):
            p = e[j] * inv
            ds = p * (wd[j] - di)
            gq = _fma(ds[..., None], K[:, :, None, j], gq)
            stv, stk = GO * p[..., None], Q * ds[..., None]
            sv, sk = np.zeros((G, H, D), f32), np.zeros((G, H, D), f32)
            for l_ in range(L):
                sv, sk = sv + stv[:, :, l_], sk + stk[:, :, l_]
            gv[:, :, j], gk[:, :, j] = sv, sk * sc
    gq = gq * sc
    B, R = q.shape[0], q.shape[1]
    un = lambda x: x.transpose(0, 2, 1, 3).reshape(G, -1, C)                # noqa: E731
    return {"o": VT._from_groups(un(o), B, R, g), "dq": VT._from_groups(un(gq), B, R, g), "dk": un(gk), "dv": un(gv)}


def emulate_layer_norm(a, b, gn, gy, w, bb, eps):
    """ln_fwd_kernel and ln_bwd_kernel's operation order in fp32: lane sums over j, the xor butterfly, the centred FMA
    variance; the backward's lane chains, per-CTA dgamma / dbeta (8 rows per warp in a chain, warps in order) and the
    fp64 sum over the CTAs."""
    a, gam, bet = a.numpy(), w.numpy(), bb.numpy()
    y = a + b.numpy() if b is not None else a
    rows, C = y.shape
    nj = C // 32
    lanes = lambda x: x.reshape(rows, nj, 32)                                # noqa: E731
    yl = lanes(y)
    s = np.zeros((rows, 32), f32)
    for j in range(nj):
        s = s + yl[:, j]
    mean = _butterfly(s) / f32(C)
    v = np.zeros((rows, 32), f32)
    for j in range(nj):
        d = yl[:, j] - mean[:, None]
        v = _fma(d, d, v)
    rstd = f32(1) / np.sqrt(_butterfly(v) / f32(C) + f32(eps))
    yh = (y - mean[:, None]) * rstd[:, None]
    res = {"y": y, "n": _fma(yh, gam, bet)}
    g = gn.numpy()
    gg = g * gam
    s1, s2 = np.zeros((rows, 32), f32), np.zeros((rows, 32), f32)
    for j in range(nj):
        s1 = s1 + lanes(gg)[:, j]
        s2 = _fma(lanes(gg)[:, j], lanes(yh)[:, j], s2)
    m1, m2 = _butterfly(s1) / f32(C), _butterfly(s2) / f32(C)
    d = rstd[:, None] * ((gg - m1[:, None]) - yh * m2[:, None])
    res["da"] = d if gy is None or b is None else gy.numpy() + d
    nparts = -(-rows // 64)
    pad = lambda x: np.concatenate([x, np.zeros((nparts * 64 - rows, C), f32)]).reshape(nparts, 8, 8, C)  # noqa: E731
    gp, yp = pad(g), pad(yh)
    dg, db = np.zeros((nparts, 8, C), f32), np.zeros((nparts, 8, C), f32)
    for i in range(8):                   # row r0 + w + 8 i of warp w
        dg, db = _fma(gp[:, i], yp[:, i], dg), db + gp[:, i]
    tg, tb = dg[:, 0], db[:, 0]
    for w_ in range(1, 8):
        tg, tb = tg + dg[:, w_], tb + db[:, w_]
    sg, sb = np.zeros(C, f64), np.zeros(C, f64)
    for p_ in range(nparts):
        sg, sb = sg + tg[p_].astype(f64), sb + tb[p_].astype(f64)
    res["dgamma"], res["dbeta"] = sg.astype(f32), sb.astype(f32)
    return res


# ---------------------------------------------------------------------------------------------------------------- CPU

# B, R, g, S, C, H, scores
CPU_ATTN = {"d16": (1, 4, 2, 3, 32, 2, "randn"), "d32_bs3": (1, 6, 2, 5, 64, 2, "randn"),
            "s1": (1, 4, 2, 1, 32, 2, "randn"), "top100": (1, 4, 2, 4, 32, 2, "top100"),
            "below100": (1, 4, 2, 4, 32, 2, "below100"), "spread": (2, 4, 2, 6, 32, 2, "spread")}
# rows, C, eps, residual b, extra dy
CPU_LN = {"c32": (65, 32, 1e-5, True, True), "c480": (130, 480, 1e-6, True, False),
          "c256_norm1": (64, 256, 1e-5, False, False), "c768": (40, 768, 1e-6, True, True)}


def _cpu_attn(name):
    B, R, g, S, C, H, kind = CPU_ATTN[name]
    return attn_inputs(B, R, g, S, C, H, kind, 3 + len(name)), g, H


def _cpu_ln(name):
    rows, C, eps, has_b, has_dy = CPU_LN[name]
    a, b, gn, gy, w, bb, const = ln_inputs(rows, C, eps, has_b, rows + C)
    return a, b, gn, gy if has_dy else None, w, bb, eps, const


@pytest.mark.parametrize("name", list(CPU_ATTN))
def test_attention_statement_equals_torch_float64(name):
    (q, k, v, up), g, H = _cpu_attn(name)
    st = attn_statement(q, k, v, up, g, H)
    ref = torch_attention(q, k, v, up, g, H, torch.float64)
    for n in ATTN_OUT:
        _pin64(ref[n], st[n], f"{name} {n}")


@pytest.mark.parametrize("name", list(CPU_LN))
def test_layer_norm_statement_equals_torch_float64(name):
    a, b, gn, gy, w, bb, eps, _ = _cpu_ln(name)
    st = ln_statement(a, b, gn, gy, w, bb, eps)
    ref = torch_layer_norm(a, b, gn, gy, w, bb, eps, torch.float64)
    for n in LN_OUT:
        _pin64(ref[n], st[n], f"{name} {n}")


@pytest.mark.parametrize("name", list(CPU_ATTN))
def test_attention_fp32_torch_and_emulation_within_bound(name):
    (q, k, v, up), g, H = _cpu_attn(name)
    st = attn_statement(q, k, v, up, g, H)
    check_all(torch_attention(q, k, v, up, g, H, torch.float32), st, ATTN_OUT, f"fp32 torch {name}")
    check_all(emulate_attention(q, k, v, up, g, H), st, ATTN_OUT, f"emulation {name}")


@pytest.mark.parametrize("name", list(CPU_LN))
def test_layer_norm_fp32_torch_and_emulation_within_bound(name):
    a, b, gn, gy, w, bb, eps, const = _cpu_ln(name)
    st = ln_statement(a, b, gn, gy, w, bb, eps)
    check_all(torch_layer_norm(a, b, gn, gy, w, bb, eps, torch.float32), st, LN_OUT, f"fp32 torch {name}")
    em = emulate_layer_norm(a, b, gn, gy, w, bb, eps)
    check_all(em, st, LN_OUT, f"emulation {name}")
    assert np.array_equal(em["n"][const], np.broadcast_to(bb.numpy(), em["n"][const].shape))


def test_score_ranges_are_what_their_cases_claim():
    """The GPU cases' input recipes at LaRa's head dim: every score below -100, and weights in expf's subnormal range."""
    q, k, _, _ = attn_inputs(1, 8, 4, 4, 64, 4, "below100", 1)
    assert float(scores64(q, k, 4, 4).max()) < -100.0
    q, k, _, _ = attn_inputs(1, 8, 4, 4, 64, 4, "spread", 1)
    s = scores64(q, k, 4, 4)
    t = s - s.max(-1, keepdim=True).values
    spread = -t.min(-1).values
    assert float(spread.min()) > 70.0 and float(spread.max()) < 100.0
    w = torch.exp(t)
    assert bool((w < 2.0 ** -126).any()) and not bool((w < 2.0 ** -149).any())


# ---------------------------------------------------------------------------------------------------------------- GPU

LARA = (3, 32, 16, 4, 256, 16)
# B, R, g, S, C, H, scores
ATTN_CASES = {
    "lara": LARA + ("randn",),
    "lara_s2": (3, 32, 16, 2, 256, 16, "randn"),
    "lara_s3": (3, 32, 16, 3, 256, 16, "randn"),
    "g8": (2, 32, 8, 32, 256, 16, "randn"),                 # 64 queries, Hs = 4
    "bs1": (2, 8, 8, 4, 256, 16, "randn"),
    "hd32": (2, 32, 16, 4, 256, 8, "randn"),
    "hd32_g8": (1, 32, 8, 24, 256, 8, "randn"),
    "bs3": (2, 12, 4, 5, 256, 16, "randn"),                 # 27 queries, Hs = 8: 216 threads, 2 head slices
    "bs5_hd32": (1, 10, 2, 6, 256, 8, "randn"),             # 125 threads, Hs = 1
    "odd_heads": (1, 16, 8, 7, 48, 3, "randn"),             # 24 threads
    "h12": (1, 16, 4, 9, 192, 12, "randn"),                 # Hs = 4, 3 slices
    "s1": (2, 32, 16, 1, 256, 16, "randn"),
    "s4096": (1, 8, 4, 4096, 64, 4, "randn"),
    "top100": (2, 32, 16, 4, 256, 16, "top100"),          # LaRa's scene shape at B = 2
    "below100": LARA + ("below100",),
    "spread": LARA + ("spread",),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ATTN_CASES))
def test_group_attention_kernels_per_element(cuda_device, name):
    from lara_b200.vol_transformer import group_attention
    B, R, g, S, C, H, kind = ATTN_CASES[name]
    q, k, v, up = attn_inputs(B, R, g, S, C, H, kind, 100 + len(name))
    ins = [t.to(cuda_device).requires_grad_(True) for t in (q, k, v)]
    o = group_attention(*ins, g, H)
    o.backward(up.to(cuda_device))
    res = {"o": _np(o), "dq": _np(ins[0].grad), "dk": _np(ins[1].grad), "dv": _np(ins[2].grad)}
    st = attn_statement(q, k, v, up, g, H)
    check_all(res, st, ATTN_OUT, f"kernels {name}")


# entry, rows, C, eps, residual b, extra dy
LN_CASES = {
    "lara_add": ("srf_add_layernorm", 3 * 32 ** 3, 256, 1e-5, True, True),
    "lara_norm": ("srf_add_layernorm", 3 * 32 ** 3, 256, 1e-6, True, False),
    "lara_norm1": ("srf_add_layernorm", 3 * 32 ** 3, 256, 1e-5, False, False),
    "c32": ("srf_add_layernorm", 1001, 32, 1e-5, True, True),
    "c480": ("srf_add_layernorm", 777, 480, 1e-5, True, True),      # nj = 15
    "c512": ("srf_add_layernorm", 777, 512, 1e-6, True, False),
    "rows0": ("srf_add_layernorm", 0, 256, 1e-5, True, True),
    "rows1": ("srf_add_layernorm", 1, 256, 1e-5, True, True),
    "rows63": ("srf_add_layernorm", 63, 256, 1e-5, True, True),
    "rows64": ("srf_add_layernorm", 64, 256, 1e-5, True, False),
    "rows65": ("srf_add_layernorm", 65, 256, 1e-6, False, False),
    "vit768": ("srf_vit_layernorm", 12 * 1025, 768, 1e-6, True, True),
    "vit768_rows1": ("srf_vit_layernorm", 1, 768, 1e-6, True, True),
    "vit768_rows777": ("srf_vit_layernorm", 777, 768, 1e-6, True, True),
    "vit384": ("srf_vit_layernorm", 12 * 1025, 384, 1e-6, True, True),
    "vit384_rows1": ("srf_vit_layernorm", 1, 384, 1e-6, True, True),
    "vit384_rows777": ("srf_vit_layernorm", 777, 384, 1e-6, True, True),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(LN_CASES))
def test_layernorm_kernels_per_element(cuda_device, name):
    from lara_b200.vol_transformer import _AddLayerNorm
    entry, rows, C, eps, has_b, has_dy = LN_CASES[name]
    a, b, gn, gy, w, bb, const = ln_inputs(rows, C, eps, has_b, rows + C)
    dev = cuda_device
    ins = [t.to(dev).clone().requires_grad_(True) if t is not None else None for t in (a, b, w, bb)]
    out = _AddLayerNorm.apply(*ins, eps, entry)
    y, n = out if has_b else (None, out)
    torch.autograd.backward([n] + ([y] if has_dy else []), [gn.to(dev)] + ([gy.to(dev)] if has_dy else []))
    res = {"n": _np(n), "da": _np(ins[0].grad), "dgamma": _np(ins[2].grad), "dbeta": _np(ins[3].grad)}
    if has_b:
        res["y"] = _np(y)
        assert torch.equal(ins[0].grad, ins[1].grad)
    st = ln_statement(a, b, gn, gy if has_dy else None, w, bb, eps)
    if not has_b:
        del st["y"]
    check_all(res, st, LN_OUT, f"{entry} {name}")
    # exactly constant rows normalise to beta, bit for bit; no rows: exact zero parameter gradients
    assert np.array_equal(res["n"][const], np.broadcast_to(bb.numpy().astype(f64), res["n"][const].shape))
    if rows == 0:
        assert not res["dgamma"].any() and not res["dbeta"].any()
