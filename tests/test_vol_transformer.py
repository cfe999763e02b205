"""LaRa's volume transformer (GroupAttBlock.forward, lightning/network.py:81-102, and VolTransformer.forward, :138-164)
on a channels-last volume, with the group cross-attention and the residual add + LayerNorms in CUDA.

* CPU: the torch restatement ``oracle.vol_transformer_torch`` is pinned bit for bit against LaRa's own
  ``GroupAttBlock`` and ``VolTransformer`` (g = R/2 and R/4, V = 3, and two alternating ``n_groups`` entries): the
  output and the gradients of x, the condition, ``pos_embed`` and every parameter under a seeded upstream gradient.
  LaRa's outputs are recorded in tests/golden/reference/test_vol_transformer.npz by record_reference:

      python tests/test_vol_transformer.py OUT_DIR LARA_CHECKOUT && cp OUT_DIR/test_vol_transformer.npz tests/golden/reference/

  The channels-last restatement equals LaRa's layout in float64 to 1e-12; the drop-in's state-dict keys and shapes
  equal LaRa's; the argument checks of the Python and C entries run without a GPU.
* GPU (TF32 off for the fp32 comparisons): one block and a 3-layer transformer against the float64 restatement,
  beside LaRa's own fp32 block on the same inputs; bit-reproducibility with the deterministic switch off and on; bf16
  autocast against LaRa's block under autocast.  The attention and LayerNorm kernels themselves, forward and backward,
  are checked element by element against a float64 statement with a bound per element in
  tests/test_vol_transformer_per_element.py.
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from helpers import fingerprint, reference_record
from test_decoder_layout import _import_reference_network

# ---- seeded parameters and inputs --------------------------------------------------------------------------------


def block_params(C, Cc, seed, prefix="", mlp_ratio=2.0):
    """A GroupAttBlock's parameters under LaRa's names, seeded (fp32, CPU)."""
    g = torch.Generator().manual_seed(seed)
    hid = int(C * mlp_ratio)

    def u(*shape, fan):
        return (torch.rand(shape, generator=g) * 2 - 1) / fan ** 0.5
    p = {}
    for n in ("norm1", "norm2", "norm3"):
        p[n + ".weight"] = 1 + 0.2 * torch.randn(C, generator=g)
        p[n + ".bias"] = 0.1 * torch.randn(C, generator=g)
    p["cross_attn.q_proj_weight"] = u(C, C, fan=C)
    p["cross_attn.k_proj_weight"] = u(C, Cc, fan=Cc)
    p["cross_attn.v_proj_weight"] = u(C, Cc, fan=Cc)
    p["cross_attn.out_proj.weight"] = u(C, C, fan=C)
    p["mlp.0.weight"], p["mlp.0.bias"] = u(hid, C, fan=C), u(hid, fan=C)
    p["mlp.3.weight"], p["mlp.3.bias"] = u(C, hid, fan=hid), u(C, fan=hid)
    p["cnn.weight"] = u(C, C, 3, 3, 3, fan=27 * C)
    return {prefix + k: v for k, v in p.items()}


def transformer_params(C, Cc, R, out_dim, layers, seed):
    g = torch.Generator().manual_seed(seed)
    p = {"pos_embed": torch.randn((1, C, R, R, R), generator=g) / C ** 0.5}
    for i in range(layers):
        p.update(block_params(C, Cc, seed + 1 + i, f"layers.{i}."))
    p["norm.weight"] = 1 + 0.2 * torch.randn(C, generator=g)
    p["norm.bias"] = 0.1 * torch.randn(C, generator=g)
    p["deconv.weight"] = (torch.rand((C, out_dim, 2, 2, 2), generator=g) * 2 - 1) / (8 * C) ** 0.5
    p["deconv.bias"] = 0.1 * torch.randn(out_dim, generator=g)
    return p


# ---- CPU: restatement vs LaRa's own code -------------------------------------------------------------------------
# C, Cc, H, B, V, R, Rc; block cases: n_group; the transformer: n_groups, layers, out_dim
CPU = dict(C=32, Cc=24, H=2, B=2, V=3, R=4, Rc=2)
BLOCK_CASES = {"block_g2": 2, "block_g1": 1}            # g = R/2 (bs 2, S = V) and R/4 (bs 4, S = 8 V)
TF_CASE = dict(n_groups=[2, 1], layers=3, out_dim=5)


def _block_inputs(name):
    c, ng = CPU, BLOCK_CASES[name]
    g = torch.Generator().manual_seed(11 + ng)
    S = c["V"] * (c["Rc"] // ng) ** 3
    x = torch.randn((c["B"], c["C"], c["R"], c["R"], c["R"]), generator=g)
    cond = torch.randn((c["B"] * ng ** 3, S, c["Cc"]), generator=g)
    up = torch.randn(x.shape, generator=g)
    return x, cond, ng, block_params(c["C"], c["Cc"], 40 + ng), up


def _tf_inputs():
    c = CPU
    g = torch.Generator().manual_seed(5)
    feats = torch.randn((c["B"], c["V"], c["Cc"], c["Rc"], c["Rc"], c["Rc"]), generator=g)
    p = transformer_params(c["C"], c["Cc"], c["R"], TF_CASE["out_dim"], TF_CASE["layers"], 60)
    up = torch.randn((c["B"], 2 * c["R"], 2 * c["R"], 2 * c["R"], TF_CASE["out_dim"]), generator=g)
    return feats, p, up


def _record(out, inputs, params):
    rec = {"out": fingerprint(out.detach().numpy())}
    rec.update({"g_" + k: fingerprint(t.grad.numpy()) for k, t in inputs.items()})
    rec.update({"g_" + k: fingerprint(t.grad.numpy()) for k, t in params.items()})
    return rec


def state_signature(sd):
    return ";".join(f"{k}:{tuple(v.shape)}" for k, v in sorted(sd.items()))


def record_reference(lara, dev):
    """LaRa's own GroupAttBlock and VolTransformer on the CPU."""
    net = _import_reference_network(lara)
    c, recs = CPU, {}
    for name in BLOCK_CASES:
        x, cond, ng, p, up = _block_inputs(name)
        blk = net.GroupAttBlock(inner_dim=c["C"], cond_dim=c["Cc"], num_heads=c["H"], eps=1e-6)
        blk.load_state_dict(p, strict=True)
        x, cond = x.requires_grad_(True), cond.requires_grad_(True)
        out = blk(x, cond, ng, c["R"] // ng)
        out.backward(up)
        recs[name] = _record(out, {"x": x, "cond": cond}, dict(blk.named_parameters()))
    feats, p, up = _tf_inputs()
    vt = net.VolTransformer(embed_dim=c["C"], image_feat_dim=c["Cc"], n_groups=TF_CASE["n_groups"], vol_low_res=c["R"],
                            vol_high_res=2 * c["R"], out_dim=TF_CASE["out_dim"], num_layers=TF_CASE["layers"],
                            num_heads=c["H"])
    vt.load_state_dict(p, strict=True)
    feats = feats.requires_grad_(True)
    out = vt(feats)
    out.backward(up)
    recs["transformer"] = _record(out, {"image_feats": feats}, dict(vt.named_parameters()))
    recs["state"] = {"signature": np.array(state_signature(vt.state_dict()))}
    return recs


@pytest.mark.parametrize("name", sorted(BLOCK_CASES))
def test_group_att_block_restatement_matches_reference_on_cpu(name):
    from oracle.vol_transformer_torch import group_att_block_torch
    x, cond, ng, p, up = _block_inputs(name)
    x, cond = x.requires_grad_(True), cond.requires_grad_(True)
    p = {k: v.requires_grad_(True) for k, v in p.items()}
    out = group_att_block_torch(x, cond, ng, CPU["R"] // ng, p, CPU["H"])
    out.backward(up)
    mine = _record(out, {"x": x, "cond": cond}, p)
    ref = reference_record("test_vol_transformer", name)
    assert sorted(mine) == sorted(ref)
    assert [k for k in mine if mine[k] != ref[k]] == []


def test_vol_transformer_restatement_matches_reference_on_cpu():
    from oracle.vol_transformer_torch import vol_transformer_torch
    feats, p, up = _tf_inputs()
    feats = feats.requires_grad_(True)
    p = {k: v.requires_grad_(True) for k, v in p.items()}
    out = vol_transformer_torch(feats, p, TF_CASE["n_groups"], CPU["H"], CPU["R"])
    assert out.is_contiguous()
    out.backward(up)
    mine = _record(out, {"image_feats": feats}, p)
    ref = reference_record("test_vol_transformer", "transformer")
    assert sorted(mine) == sorted(ref)
    assert [k for k in mine if mine[k] != ref[k]] == []


def test_channels_last_restatement_equals_laras_layout_in_float64():
    from oracle.vol_transformer_torch import (cond_blocks_torch, group_att_block_cl, group_att_block_torch,
                                              vol_transformer_cl, vol_transformer_torch)
    c = CPU
    for name in BLOCK_CASES:
        x, cond, ng, p, _ = _block_inputs(name)
        p = {k: v.double() for k, v in p.items()}
        ref = group_att_block_torch(x.double(), cond.double(), ng, c["R"] // ng, p, c["H"])
        cl = group_att_block_cl(x.double().permute(0, 2, 3, 4, 1), cond.double(), ng, p, c["H"])
        assert float((cl.permute(0, 4, 1, 2, 3) - ref).abs().max()) <= 1e-12 * float(ref.abs().max()), name
    feats, p, _ = _tf_inputs()
    feats, p = feats.double(), {k: v.double() for k, v in p.items()}
    ref = vol_transformer_torch(feats, p, TF_CASE["n_groups"], c["H"], c["R"])
    cl = vol_transformer_cl([cond_blocks_torch(feats, g) for g in TF_CASE["n_groups"]], p, TF_CASE["n_groups"], c["H"],
                            c["B"])
    assert float((cl - ref).abs().max()) <= 1e-12 * float(ref.abs().max())


def _drop_in(C=CPU["C"], Cc=CPU["Cc"], H=CPU["H"], R=CPU["R"], n_groups=None, layers=TF_CASE["layers"],
             out_dim=TF_CASE["out_dim"]):
    from lara_b200.vol_transformer import VolTransformer
    return VolTransformer(embed_dim=C, image_feat_dim=Cc, n_groups=n_groups or TF_CASE["n_groups"], vol_low_res=R,
                          vol_high_res=2 * R, out_dim=out_dim, num_layers=layers, num_heads=H)


def test_vol_transformer_state_dict_matches_laras():
    vt = _drop_in()
    ref = reference_record("test_vol_transformer", "state")
    assert state_signature(vt.state_dict()) == ref["signature"]
    _, p, _ = _tf_inputs()
    vt.load_state_dict(p, strict=True)


# ---- CPU: argument checks ----------------------------------------------------------------------------------------
def test_group_att_block_constructor_rejects_unsupported_sizes():
    from lara_b200.vol_transformer import GroupAttBlock, VolTransformer
    for C, Cc, H in ((48, 24, 3), (32, 24, 4), (32, 24, 3), (544, 24, 17), (32, 32, 2), (32, 0, 2)):
        with pytest.raises(ValueError, match="GroupAttBlock"):
            GroupAttBlock(C, Cc, H)
    for ng in ([3], [], [0]):
        with pytest.raises(ValueError, match="VolTransformer"):
            VolTransformer(32, 24, ng, 4, 8, 5, 1, 2)


def test_vol_transformer_rejects_bad_inputs_before_any_launch():
    from lara_b200.vol_transformer import add_layer_norm, group_attention
    vt = _drop_in()
    with pytest.raises(RuntimeError, match="VolTransformer.forward: need one condition tensor"):
        vt([torch.zeros(16, 3, 24)])
    with pytest.raises(RuntimeError, match="must be \\[B,V,C,D,D,D\\]"):
        vt(torch.zeros(2, 3, 24, 2, 2))
    with pytest.raises(RuntimeError, match="multiple of every n_groups"):
        vt(torch.zeros(2, 3, 24, 3, 3, 3))
    with pytest.raises(RuntimeError, match="disagree on the batch size"):
        vt([torch.zeros(16, 3, 24), torch.zeros(1, 24, 24)])
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        vt(torch.zeros(2, 3, 24, 2, 2, 2))
    blk = vt.layers[0]
    with pytest.raises(RuntimeError, match="group_axis \\* block_size"):
        blk(torch.zeros(2, 32, 4, 4, 4), torch.zeros(16, 3, 24), 2, 1)
    with pytest.raises(RuntimeError, match="cond must be"):
        blk(torch.zeros(2, 32, 4, 4, 4), torch.zeros(16, 3, 23), 2, 2)
    with pytest.raises(RuntimeError, match="Float"):
        add_layer_norm(torch.zeros(4, 32, dtype=torch.float64), None, blk.norm1)
    with pytest.raises(RuntimeError, match="multiple of 32 up to 512"):
        add_layer_norm(torch.zeros(4, 48), None, torch.nn.LayerNorm(48))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        add_layer_norm(torch.zeros(4, 32), torch.zeros(4, 32), blk.norm1)
    q, kv = torch.zeros(1, 4, 4, 4, 32), torch.zeros(8, 3, 32)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        group_attention(q, kv, kv, 2, 2)
    for args, msg in (((torch.zeros(1, 4, 4, 3, 32), kv, kv, 2, 2), "q must be"),
                      ((q, kv, kv, 3, 2), "n_group"), ((q, kv, kv, 2, 4), "head dim"),
                      ((q, kv[:4], kv[:4], 2, 2), "k and v"), ((q, kv, kv[:, :2], 2, 2), "k and v")):
        with pytest.raises(RuntimeError, match=msg):
            group_attention(*args)


LARA_ATTN = [3, 32, 16, 4, 256, 16]      # B, R, g, S, C, H


def test_vol_transformer_c_entries_reject_bad_arguments_before_any_launch(lib):
    P = ctypes.c_void_p(256)             # never dereferenced: the checks come before any CUDA call
    for i, bad in ((0, 0), (1, 0), (2, 0), (2, 3), (1, 2048), (3, 0), (3, 4097), (4, 48), (5, 5), (5, 0), (4, 128),
                   (5, 4)):
        a = list(LARA_ATTN)
        a[i] = bad
        assert lib.srf_group_attn_forward(None, *a, P, P, P, P) != 0
        assert b"srf_group_attn_forward: bad sizes" in lib.srf_last_error()
        assert lib.srf_group_attn_backward(None, *a, P, P, P, P, P, P, P) != 0
        assert b"srf_group_attn_backward: bad sizes" in lib.srf_last_error()
    a = [1, 32, 2, 4, 256, 16]           # bs = 16: 4096 queries x 16 > 4096
    assert lib.srf_group_attn_forward(None, *a, P, P, P, P) != 0
    assert b"(R/g)^3 * C/H" in lib.srf_last_error()
    for k in range(4):
        ptrs = [P] * 4
        ptrs[k] = None
        assert lib.srf_group_attn_forward(None, *LARA_ATTN, *ptrs) != 0
        assert b"null pointer" in lib.srf_last_error()
    for k in range(7):
        ptrs = [P] * 7
        ptrs[k] = ctypes.c_void_p(260)
        assert lib.srf_group_attn_backward(None, *LARA_ATTN, *ptrs) != 0
        assert b"16-byte aligned" in lib.srf_last_error()
    size = ctypes.c_size_t()
    for rows, C, eps in ((-1, 256, 1e-5), (8, 48, 1e-5), (8, 0, 1e-5), (8, 544, 1e-5), (8, 256, 0.0),
                         (8, 256, float("nan"))):
        assert lib.srf_add_layernorm_forward(None, rows, C, eps, P, P, P, P, P, P) != 0
        assert b"srf_add_layernorm_forward: bad" in lib.srf_last_error()
        assert lib.srf_add_layernorm_backward(None, rows, C, eps, P, P, P, P, P, P, P, P) != 0
        assert b"srf_add_layernorm_backward: bad" in lib.srf_last_error()
    assert lib.srf_add_layernorm_workspace_bytes(8, 48, ctypes.byref(size)) != 0
    assert lib.srf_add_layernorm_workspace_bytes(8, 256, None) != 0
    assert lib.srf_add_layernorm_workspace_bytes(100, 256, ctypes.byref(size)) == 0 and size.value >= 2 * 2 * 256 * 4
    assert lib.srf_add_layernorm_forward(None, 8, 256, 1e-5, P, P, P, P, None, P) != 0
    assert b"null y with a residual b" in lib.srf_last_error()
    assert lib.srf_add_layernorm_forward(None, 8, 256, 1e-5, None, None, P, P, None, P) != 0
    assert b"null pointer" in lib.srf_last_error()
    assert lib.srf_add_layernorm_backward(None, 8, 256, 1e-5, P, P, P, None, ctypes.c_void_p(264), P, P, P) != 0
    assert b"workspace must be 256-byte aligned" in lib.srf_last_error()
    assert lib.srf_add_layernorm_backward(None, 8, 256, 1e-5, P, P, P, None, P, P, None, P) != 0
    assert b"null gradient pointer" in lib.srf_last_error()


# ---- GPU ----------------------------------------------------------------------------------------------------------
@pytest.fixture
def no_tf32():
    m, c = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = m, c


def _err(a, ref):
    a, ref = a.double(), ref.double()
    m = float(ref.abs().max()) if ref.numel() else 0.0
    return float((a - ref).abs().max()) / (m if m > 0 else 1.0) if ref.numel() else 0.0


LARA_V4 = (3, 32, 16, 4, 256, 16)       # B, R, g, S, C, H


def _attn_inputs(dev):
    B, R, g, S, C, H = LARA_V4
    gen = torch.Generator().manual_seed(24)
    q = torch.randn((B, R, R, R, C), generator=gen)
    k = torch.randn((B * g ** 3, S, C), generator=gen)
    v = torch.randn((B * g ** 3, S, C), generator=gen)
    up = torch.randn(q.shape, generator=gen)
    return [t.to(dev) for t in (q, k, v, up)], g, H


# a reduced LaRa: C, Cc, H, B, V, R, Rc, n_groups
MODEL = dict(C=64, Cc=80, H=4, B=2, V=3, R=16, Rc=8, n_groups=[8, 4])


def _model_inputs(dev, layers):
    c = MODEL
    gen = torch.Generator().manual_seed(3)
    feats = torch.randn((c["B"], c["V"], c["Cc"], c["Rc"], c["Rc"], c["Rc"]), generator=gen)
    p = transformer_params(c["C"], c["Cc"], c["R"], 16, layers, 90)
    return feats.to(dev), {k: v.to(dev) for k, v in p.items()}


def _grads_vs(mine, ref):
    return {k: _err(mine[k], ref[k]) for k in ref}


def _run_lara_block(x, cond, p):
    from oracle.vol_transformer_torch import group_att_block_torch
    c = MODEL
    ng = c["n_groups"][0]
    x = x.clone().requires_grad_(True)
    cond = cond.clone().requires_grad_(True)
    p = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    out = group_att_block_torch(x, cond, ng, c["R"] // ng, p, c["H"])
    return out, x, cond, p


@pytest.mark.gpu
def test_group_att_block_matches_float64_beside_laras_fp32_block(cuda_device, no_tf32):
    from lara_b200.vol_transformer import GroupAttBlock
    from oracle.vol_transformer_torch import cond_blocks_torch
    c, dev = MODEL, cuda_device
    feats, tp = _model_inputs(dev, 1)
    p = {k[len("layers.0."):]: v for k, v in tp.items() if k.startswith("layers.0.")}
    ng = c["n_groups"][0]
    gen = torch.Generator().manual_seed(8)
    x = torch.randn((c["B"], c["C"], c["R"], c["R"], c["R"]), generator=gen).to(dev)
    cond = cond_blocks_torch(feats, ng)
    up = torch.randn(x.shape, generator=gen).to(dev)
    res = {}
    for arm in ("f64", "lara", "drop_in"):
        if arm == "drop_in":
            blk = GroupAttBlock(c["C"], c["Cc"], c["H"]).to(dev)
            blk.load_state_dict(p, strict=True)
            xi, ci = x.clone().requires_grad_(True), cond.clone().requires_grad_(True)
            out = blk(xi, ci, ng, c["R"] // ng)
            assert out.is_contiguous(memory_format=torch.channels_last_3d)
            out.backward(up)
            res[arm] = {"out": out.detach(), "x": xi.grad, "cond": ci.grad,
                        **{k: t.grad for k, t in blk.named_parameters()}}
        else:
            cast = (lambda t: t.double()) if arm == "f64" else (lambda t: t)
            out, xi, ci, pi = _run_lara_block(cast(x), cast(cond), {k: cast(v) for k, v in p.items()})
            out.backward(cast(up))
            res[arm] = {"out": out.detach(), "x": xi.grad, "cond": ci.grad, **{k: t.grad for k, t in pi.items()}}
    lara, mine = _grads_vs(res["lara"], res["f64"]), _grads_vs(res["drop_in"], res["f64"])
    print("block worst error: drop-in", f"{max(mine.values()):.2e}", "LaRa fp32", f"{max(lara.values()):.2e}")
    bad = {k: (f"{mine[k]:.2e}", f"{lara[k]:.2e}") for k in mine if not mine[k] <= max(2 * lara[k], 1e-6)}
    assert bad == {}, bad


@pytest.mark.gpu
def test_vol_transformer_matches_float64_beside_laras_fp32_transformer(cuda_device, no_tf32):
    from oracle.vol_transformer_torch import vol_transformer_torch
    c, dev, layers = MODEL, cuda_device, 3
    feats, p = _model_inputs(dev, layers)
    up = torch.randn((c["B"], 2 * c["R"], 2 * c["R"], 2 * c["R"], 16), generator=torch.Generator().manual_seed(4))
    up = up.to(dev)
    res = {}
    for arm in ("f64", "lara", "drop_in", "drop_in_list"):
        cast = (lambda t: t.double()) if arm == "f64" else (lambda t: t)
        fi = cast(feats).clone().requires_grad_(True)
        if arm.startswith("drop_in"):
            vt = _drop_in(c["C"], c["Cc"], c["H"], c["R"], c["n_groups"], layers, 16).to(dev)
            vt.load_state_dict(p, strict=True)
            if arm == "drop_in":
                out = vt(fi)
            else:
                from oracle.vol_transformer_torch import cond_blocks_torch
                out = vt([cond_blocks_torch(fi, g) for g in c["n_groups"]])
            named = dict(vt.named_parameters())
        else:
            named = {k: cast(v).clone().requires_grad_(True) for k, v in p.items()}
            out = vol_transformer_torch(fi, named, c["n_groups"], c["H"], c["R"])
        assert out.is_contiguous() and out.shape == up.shape
        out.backward(cast(up))
        res[arm] = {"out": out.detach(), "image_feats": fi.grad, **{k: t.grad for k, t in named.items()}}
    lara = _grads_vs(res["lara"], res["f64"])
    for arm in ("drop_in", "drop_in_list"):
        mine = _grads_vs(res[arm], res["f64"])
        print(arm, "transformer worst error", f"{max(mine.values()):.2e}", "LaRa fp32", f"{max(lara.values()):.2e}")
        bad = {k: (f"{mine[k]:.2e}", f"{lara[k]:.2e}") for k in mine if not mine[k] <= max(2 * lara[k], 1e-6)}
        assert bad == {}, (arm, bad)


@pytest.mark.gpu
def test_vol_transformer_kernels_are_bit_reproducible_with_the_deterministic_switch_off_and_on(cuda_device):
    from lara_b200.vol_transformer import add_layer_norm, group_attention
    dev = cuda_device
    (q, k, v, up), g, H = _attn_inputs(dev)
    rows = q.numel() // q.shape[-1]
    a, b = q.view(rows, -1), up.view(rows, -1)
    norm = torch.nn.LayerNorm(256).to(dev)

    def run():
        ins = [t.clone().requires_grad_(True) for t in (q, k, v, a, b)]
        o = group_attention(*ins[:3], g, H)
        y, n = add_layer_norm(ins[3], ins[4], norm)
        norm.zero_grad(set_to_none=True)
        torch.autograd.backward([o, n, y], [up, b, a])
        return [o.detach(), y.detach(), n.detach()] + [t.grad for t in ins] + [norm.weight.grad, norm.bias.grad]
    runs = []
    was = torch.are_deterministic_algorithms_enabled()
    try:
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            runs += [run(), run()]
    finally:
        torch.use_deterministic_algorithms(was)
    for r in runs[1:]:
        assert all(torch.equal(x, y) for x, y in zip(runs[0], r))


@pytest.mark.gpu
def test_group_att_block_under_bf16_autocast_against_laras(cuda_device):
    from lara_b200.vol_transformer import GroupAttBlock
    from oracle.vol_transformer_torch import cond_blocks_torch
    c, dev = MODEL, cuda_device
    feats, tp = _model_inputs(dev, 1)
    p = {k[len("layers.0."):]: v for k, v in tp.items() if k.startswith("layers.0.")}
    ng = c["n_groups"][0]
    x = torch.randn((c["B"], c["C"], c["R"], c["R"], c["R"]), generator=torch.Generator().manual_seed(2)).to(dev)
    cond = cond_blocks_torch(feats, ng)
    blk = GroupAttBlock(c["C"], c["Cc"], c["H"]).to(dev)
    blk.load_state_dict(p, strict=True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        mine = blk(x, cond, ng, c["R"] // ng)
        lara = _run_lara_block(x, cond, p)[0]
    with torch.no_grad():
        ref = _run_lara_block(x.double(), cond.double(), {k: v.double() for k, v in p.items()})[0]
    mine, lara = mine.detach(), lara.detach()
    e_mine, e_lara, e_between = _err(mine.float(), ref), _err(lara.float(), ref), _err(mine.float(), lara.float())
    print(f"bf16 autocast: drop-in {e_mine:.2e}, LaRa {e_lara:.2e} from float64; between them {e_between:.2e}")
    # LaRa's block returns bf16 here (its closing einsum autocasts); the drop-in's fused LayerNorm keeps fp32
    assert lara.dtype == torch.bfloat16 and mine.dtype == torch.float32
    assert e_mine <= max(2 * e_lara, 1e-2)


if __name__ == "__main__":
    # python tests/test_vol_transformer.py OUT_DIR LARA_CHECKOUT: record LaRa's outputs, as
    # tests/golden/make_reference_records.py does for the other modules
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_reference_records import save
    out_dir, lara = sys.argv[1:3]
    os.makedirs(out_dir, exist_ok=True)
    save(out_dir, "test_vol_transformer", record_reference(lara, "cpu"))
