"""Coarse-pass decoder head (Decoder.forward_coarse, lightning/network.py:259-278, and get_offseted_pt, :425-429).

* CPU: the torch restatement ``oracle.coarse_head_torch`` is pinned bit for bit against LaRa's own ``Decoder`` +
  ``Network.get_offseted_pt`` with seeded non-zero biases and a seeded upstream gradient on all five outputs: values,
  dL/dfeats and the six parameter gradients, for the offset form and the centers form.  LaRa's side is recorded in
  tests/golden/reference/test_coarse_head.npz by record_reference:

      python tests/test_coarse_head.py OUT_DIR LARA_CHECKOUT && cp OUT_DIR/test_coarse_head.npz tests/golden/reference/

  ``CoarseHead``'s state-dict keys and shapes equal the recorded ones of LaRa's ``mlp_coarse``; the argument checks of
  the Python entries and of the C entries run without a GPU.
* GPU: the kernels against the float64 restatement on the same fp32 inputs (every output element within 1e-5 of its
  tensor's float64 maximum; gradients likewise, with the ReLU decisions that fp32 cannot resolve accounted for),
  bit-reproducibility with the deterministic switch off and on, bf16 autocast, and a render -> loss chain.
"""
import ctypes
import os
import sys
import types

import numpy as np
import pytest
import torch

from helpers import fingerprint, reference_record
from test_decoder_layout import _import_reference_network

PARAM_NAMES = ("mlp_coarse.0.weight", "mlp_coarse.0.bias", "mlp_coarse.2.weight", "mlp_coarse.2.bias",
               "mlp_coarse.4.weight", "mlp_coarse.4.bias")
OUT_NAMES = ("first", "sh", "scaling", "rotation", "opacity")
TOL = 1e-5
OPACITY_SHIFT, SCALING_SHIFT = -2.1792, -4.2           # LaRa's coarse-pass shifts
LARA_HALF_CELL = 0.5 * 0.5 / 32                         # 0.5 * scene_size / n_offset_groups


def random_params(D, K, S, seed, dtype=torch.float32, bias=0.1):
    """The six mlp_coarse parameters, seeded, at the scale of LaRa's xavier initialisation, with non-zero biases."""
    g = torch.Generator().manual_seed(seed)
    O = K * (10 + S)

    def u(o, i):
        return ((torch.rand((o, i), generator=g) * 2 - 1) * (6.0 / (o + i)) ** 0.5).to(dtype)
    return [u(D, D), (bias * torch.randn(D, generator=g)).to(dtype), u(D, D), (bias * torch.randn(D, generator=g)).to(dtype),
            u(O, D), (bias * torch.randn(O, generator=g)).to(dtype)]


def state_signature(module_or_sd):
    sd = module_or_sd if isinstance(module_or_sd, dict) else module_or_sd.state_dict()
    return ";".join(f"{k}:{tuple(v.shape)}" for k, v in sorted(sd.items()))


# ---- CPU: restatement vs LaRa's own code ----------------------------------------------------------------------
B_CPU, R_CPU, D_CPU, K_CPU, S_CPU = 2, 6, 80, 2, 12       # feats [2, 6, 6, 6, 80]
N_CPU = R_CPU ** 3


def _cpu_case():
    g = torch.Generator().manual_seed(31)
    feats = torch.randn((B_CPU, R_CPU, R_CPU, R_CPU, D_CPU), generator=g)
    centers = torch.rand((1, N_CPU, 3), generator=g) - 0.5
    G = N_CPU * K_CPU
    ups = [torch.randn(s, generator=g) for s in ((B_CPU, G, 3), (B_CPU, G, S_CPU // 3, 3), (B_CPU, G, 2),
                                                  (B_CPU, G, 4), (B_CPU, G, 1))]
    return feats, centers, ups


def _record(outs, feats, params):
    rec = {n: fingerprint(o.detach().numpy()) for n, o in zip(OUT_NAMES, outs)}
    rec["g_feats"] = fingerprint(feats.grad.numpy())
    rec.update({"g_" + k: fingerprint(p.grad.numpy()) for k, p in zip(PARAM_NAMES, params)})
    return rec


def record_reference(lara, dev):
    """LaRa's own Decoder.forward_coarse (+ Network.get_offseted_pt) on the CPU."""
    net = _import_reference_network(lara)
    out = {}
    for form in ("offset", "centers"):
        dec = net.Decoder(D_CPU, S_CPU, 2, 4, 1, K=K_CPU)
        dec.load_state_dict(dict(zip(PARAM_NAMES, random_params(D_CPU, K_CPU, S_CPU, 5))), strict=False)
        feats, centers, ups = _cpu_case()
        feats.requires_grad_(True)
        outs = list(dec.forward_coarse(feats, OPACITY_SHIFT, SCALING_SHIFT))
        if form == "centers":
            fake = types.SimpleNamespace(scene_size=0.5, n_offset_groups=R_CPU, group_centers=centers)
            outs[0] = net.Network.get_offseted_pt(fake, outs[0], K_CPU)
        torch.autograd.backward(outs, ups)
        params = [dict(dec.named_parameters())[k] for k in PARAM_NAMES]
        out[form] = _record(outs, feats, params)
        coarse = {k: v for k, v in dec.state_dict().items() if k.startswith("mlp_coarse")}
        out["state"] = {"signature": np.array(state_signature(coarse))}
    return out


@pytest.mark.parametrize("form", ["offset", "centers"])
def test_coarse_head_restatement_matches_reference_on_cpu(form):
    from oracle.coarse_head_torch import coarse_head_torch
    feats, centers, ups = _cpu_case()
    feats.requires_grad_(True)
    params = [p.requires_grad_(True) for p in random_params(D_CPU, K_CPU, S_CPU, 5)]
    gc = centers if form == "centers" else None
    outs = coarse_head_torch(feats, params, K_CPU, S_CPU, OPACITY_SHIFT, SCALING_SHIFT, gc, 0.5 * 0.5 / R_CPU)
    torch.autograd.backward(outs, ups)
    mine = _record(outs, feats, params)
    ref = reference_record("test_coarse_head", form)
    assert sorted(mine) == sorted(ref)
    assert [k for k in mine if mine[k] != ref[k]] == []


def test_coarse_head_state_dict_matches_laras_mlp_coarse():
    from lara_b200 import CoarseHead
    head = CoarseHead(D_CPU, S_CPU, K_CPU)
    assert state_signature(head) == reference_record("test_coarse_head", "state")["signature"]
    assert sorted(k for k, _ in head.named_parameters()) == sorted(PARAM_NAMES)
    assert all(float(p.detach().abs().sum()) == 0 for k, p in head.named_parameters() if k.endswith("bias"))


# ---- CPU: argument checks ----------------------------------------------------------------------------------------
def test_coarse_head_constructor_rejects_unsupported_sizes():
    from lara_b200 import CoarseHead
    for D, S, K in ((8, 12, 2), (24, 12, 2), (144, 12, 2), (80, 9, 2), (80, 75, 2), (80, 12, 0), (80, 12, 5)):
        with pytest.raises(ValueError, match="CoarseHead"):
            CoarseHead(D, S, K)


def test_coarse_head_rejects_bad_inputs_before_any_launch():
    from lara_b200 import CoarseHead
    head = CoarseHead(16, 12, 2)
    with pytest.raises(RuntimeError, match="CoarseHead.forward_coarse"):
        head.forward_coarse(torch.zeros((2, 5, 8)), 0.0, 0.0)
    with pytest.raises(RuntimeError, match="Float"):
        head.forward_coarse(torch.zeros((2, 5, 16), dtype=torch.float64), 0.0, 0.0)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        head.forward_coarse(torch.zeros((2, 5, 16)), 0.0, 0.0)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        head.gaussians(torch.zeros((2, 5, 16)), torch.zeros((5, 3)), 0.0, 0.0, 0.1)
    with pytest.raises(RuntimeError, match="group_centers is required"):
        head.gaussians(torch.zeros((2, 5, 16)), None, 0.0, 0.0, 0.1)


def test_coarse_head_c_entries_reject_bad_sizes_before_any_launch(lib):
    P = ctypes.c_void_p(256)           # never dereferenced: the checks come before any CUDA call
    w = [P] * 6
    size = ctypes.c_size_t()
    bad = [(8, 4, 8, 2, 12), (8, 4, 24, 2, 12), (8, 4, 144, 2, 12), (8, 4, 16, 0, 12), (8, 4, 16, 5, 12),
           (8, 4, 16, 2, 9), (8, 4, 16, 2, 75), (-4, 4, 16, 2, 12), (8, 0, 16, 2, 12), (9, 4, 16, 2, 12),
           (2 ** 30, 1, 16, 4, 12)]
    for rows, N, D, K, S in bad:
        assert lib.srf_coarse_head_forward(None, rows, N, D, K, S, 0.0, 0.0, 0.1, P, None, *w, P, P, P, P, P) != 0
        assert b"srf_coarse_head_forward: bad sizes" in lib.srf_last_error()
        assert lib.srf_coarse_head_backward(None, rows, N, D, K, S, 0.1, P, None, *w, P, P, P, P, P, P, P, *w) != 0
        assert b"srf_coarse_head_backward: bad sizes" in lib.srf_last_error()
        if N == 4 and rows % 4 == 0 and rows >= 0:
            assert lib.srf_coarse_head_workspace_bytes(rows, D, K, S, ctypes.byref(size)) != 0
            assert b"srf_coarse_head_workspace_bytes: bad sizes" in lib.srf_last_error()


def test_coarse_head_c_entries_reject_null_pointers_before_any_launch(lib):
    P = ctypes.c_void_p(256)
    w = [P] * 6
    for k in range(6):
        nulled = list(w)
        nulled[k] = None
        assert lib.srf_coarse_head_forward(None, 8, 4, 16, 2, 12, 0.0, 0.0, 0.1, P, None, *nulled, P, P, P, P, P) != 0
        assert b"null weight pointer" in lib.srf_last_error()
        assert lib.srf_coarse_head_backward(None, 8, 4, 16, 2, 12, 0.1, P, None, *nulled, P, P, P, P, P, P, P, *w) != 0
        assert b"null weight pointer" in lib.srf_last_error()
        assert lib.srf_coarse_head_backward(None, 8, 4, 16, 2, 12, 0.1, P, None, *w, P, P, P, P, P, P, P, *nulled) != 0
        assert b"null weight-gradient pointer" in lib.srf_last_error()
    assert lib.srf_coarse_head_forward(None, 8, 4, 16, 2, 12, 0.0, 0.0, 0.1, None, None, *w, P, P, P, P, P) != 0
    assert b"null input pointer" in lib.srf_last_error()
    for k in range(5):
        outs = [P] * 5
        outs[k] = None
        assert lib.srf_coarse_head_forward(None, 8, 4, 16, 2, 12, 0.0, 0.0, 0.1, P, None, *w, *outs) != 0
        assert b"null output pointer" in lib.srf_last_error()
    assert lib.srf_coarse_head_forward(None, 8, 4, 16, 2, 12, 0.0, 0.0, 0.1, ctypes.c_void_p(260), None, *w,
                                       P, P, P, P, P) != 0
    assert b"16-byte aligned" in lib.srf_last_error()
    assert lib.srf_coarse_head_backward(None, 8, 4, 16, 2, 12, 0.1, P, None, *w, P, P, P, P, P,
                                        ctypes.c_void_p(264), P, *w) != 0
    assert b"workspace must be 256-byte aligned" in lib.srf_last_error()
    assert lib.srf_coarse_head_backward(None, 8, 4, 16, 2, 12, 0.1, P, None, *w, P, P, P, P, P, P, None, *w) != 0
    assert b"null feats or dL_dfeats" in lib.srf_last_error()
    # rows == 0: nothing to read or write in the forward
    assert lib.srf_coarse_head_forward(None, 0, 4, 16, 2, 12, 0.0, 0.0, 0.1, None, None, *w, None, None, None, None,
                                       None) == 0


# ---- GPU ----------------------------------------------------------------------------------------------------------
def _head(D, K, S, params, dev):
    from lara_b200 import CoarseHead
    head = CoarseHead(D, S, K).to(dev)
    with torch.no_grad():
        for p, v in zip(head._params(), params):
            p.copy_(v)
    return head


def _run_kernel(head, feats, gc, ups, half_cell):
    x = feats.clone().requires_grad_(True)
    head.zero_grad(set_to_none=True)
    if gc is None:
        outs = head.forward_coarse(x, OPACITY_SHIFT, SCALING_SHIFT)
    else:
        outs = head.gaussians(x, gc, OPACITY_SHIFT, SCALING_SHIFT, half_cell)
    torch.autograd.backward(outs, ups)
    return [o.detach() for o in outs], x.grad, [p.grad for p in head._params()]


def _run_torch(feats, gc, ups, params, K, S, half_cell):
    from oracle.coarse_head_torch import coarse_head_torch
    x = feats.clone().requires_grad_(True)
    ps = [p.detach().clone().requires_grad_(True) for p in params]
    outs = coarse_head_torch(x, ps, K, S, OPACITY_SHIFT, SCALING_SHIFT, gc, half_cell)
    torch.autograd.backward(outs, ups)
    return [o.detach() for o in outs], x.grad, [p.grad for p in ps]


def _undecided(x, params):
    """Per row: whether a hidden unit's ReLU decision is within fp32 reach (|z| <= 1e-5 (sum |w h| + |b|)); and the
    number of such units."""
    w0, b0, w1, b1 = (p.double() for p in params[:4])
    und = torch.zeros(x.shape[0], dtype=torch.bool, device=x.device)
    units = 0
    h = x
    for w, b in ((w0, b0), (w1, b1)):
        z = h @ w.T + b
        close = z.abs() <= TOL * (h.abs() @ w.abs().T + b.abs())
        und |= close.any(1)
        units += int(close.sum())
        h = torch.relu(z)
    return und, units


def _slack(x, params, ups_rows, und):
    """Per parameter tensor: the summed magnitude of the undecided rows' contributions (|dz| |h|^T, |dz|)."""
    if not bool(und.any()):
        return [0.0] * 6
    xr = x[und].double().requires_grad_(False)
    w0, b0, w1, b1, w2, b2 = (p.double() for p in params)
    z0 = xr @ w0.T + b0
    h1 = torch.relu(z0)
    z1 = h1 @ w1.T + b1
    h2 = torch.relu(z1)
    dy = ups_rows[und].double()
    dz1 = (dy @ w2) * (z1 > 0)
    dz0 = (dz1 @ w1) * (z0 > 0)
    out = []
    for dz, h in ((dz0, xr), (dz1, h1), (dy, h2)):
        out += [(dz.abs().T @ h.abs()), dz.abs().sum(0)]
    return out


def _dy_rows(feats, params, gc, ups, K, S, half_cell):
    """dL/dy per row (float64): the layout's vjp of the upstream gradients."""
    from oracle.coarse_head_torch import mlp_coarse_torch
    from oracle.torch_restatements import decoder_layout_torch
    D = feats.shape[-1]
    x = feats.reshape(-1, D).double()
    y = mlp_coarse_torch(x, [p.double() for p in params]).detach().requires_grad_(True)
    B = feats.shape[0]
    yb = y.view(B, -1, y.shape[-1])
    if gc is None:
        from oracle.coarse_head_torch import coarse_head_torch
        outs = coarse_head_torch(yb, [torch.eye(y.shape[-1], dtype=torch.float64, device=y.device),
                                      torch.zeros(y.shape[-1], dtype=torch.float64, device=y.device)] * 3,
                                 K, S, OPACITY_SHIFT, SCALING_SHIFT)
    else:
        outs = decoder_layout_torch(yb, gc.double(), K, S, OPACITY_SHIFT, SCALING_SHIFT, half_cell)
    torch.autograd.backward(outs, [u.double() for u in ups])
    return y.grad


def _rel(a, ref):
    a, ref = a.double(), ref.double()
    if ref.numel() == 0:
        return 0.0
    m = float(ref.abs().max())
    return float((a - ref).abs().max()) / (m if m > 0 else 1.0)


def _accuracy_case(dev, B, N, D, K, S, form="centers", seed=0, scale=1.0, bias=0.1, logit=None, strided=False):
    g = torch.Generator().manual_seed(seed + N)
    params = random_params(D, K, S, seed, bias=bias)
    if logit is not None:              # offset logits of +-logit: rows of W2 for offsets set to give |y| ~ logit
        C = 10 + S
        for k in range(K):
            params[4][k * C:k * C + 3] *= 0.0
            params[5][k * C:k * C + 3] = torch.tensor([logit, -logit, logit])
    feats = (torch.randn((B, N, D), generator=g) * scale).to(dev)
    if strided:                        # [B, D, N] in memory, seen as [B, N, D]
        feats = feats.transpose(1, 2).contiguous().transpose(1, 2)
        assert not feats.is_contiguous()
    gc = (torch.rand((N, 3), generator=g) - 0.5).to(dev) if form == "centers" else None
    half_cell = LARA_HALF_CELL
    G = N * K
    ups = [torch.randn(s, generator=g).to(dev) for s in ((B, G, 3), (B, G, S // 3, 3), (B, G, 2), (B, G, 4),
                                                          (B, G, 1))]
    params = [p.to(dev) for p in params]
    head = _head(D, K, S, params, dev)
    mine = _run_kernel(head, feats, gc, ups, half_cell)
    f64 = _run_torch(feats.double(), None if gc is None else gc.double(), [u.double() for u in ups],
                     [p.double() for p in params], K, S, half_cell)
    bad = []
    for name, a, b in zip(OUT_NAMES, mine[0], f64[0]):
        assert a.shape == b.shape and a.is_contiguous() and a.dtype == torch.float32, name
        if not _rel(a, b) <= TOL:
            bad.append(f"{name}: {_rel(a, b):.2e}")
    x = feats.reshape(-1, D)
    und, units = _undecided(x.double(), params)
    n_und = int(und.sum())
    rows = x.shape[0]
    # each row has 2 D hidden units; at LaRa's size about 6e-5 of them are undecided, which puts ~0.7 % of the rows
    # out of the per-row check (DESIGN §3.20)
    assert units <= 1e-4 * 2 * D * rows, f"{units} undecided hidden units in {rows} rows"
    print(f"[coarse_head] B={B} N={N} D={D} K={K} sh={S} {form}: {n_und} of {rows} rows with an undecided ReLU "
          f"({units} units) excluded from the dL/dfeats check")
    gx, gx64 = mine[1].reshape(-1, D), f64[1].reshape(-1, D)
    keep = ~und
    m = float(gx64.abs().max()) if gx64.numel() else 0.0
    if keep.any() and m > 0:
        e = float((gx[keep].double() - gx64[keep]).abs().max()) / m
        if not e <= TOL:
            bad.append(f"g_feats: {e:.2e} ({n_und} undecided rows excluded)")
    slack = _slack(x, params, _dy_rows(feats, params, gc, ups, K, S, half_cell), und) if n_und else [0.0] * 6
    for name, a, b, s in zip(PARAM_NAMES, mine[2], f64[2], slack):
        m = float(b.abs().max()) if b.numel() else 0.0
        lim = TOL * (m if m > 0 else 1.0) + (s if isinstance(s, float) else s)
        over = (a.double() - b).abs() - lim
        if float(over.max()) > 0:
            bad.append(f"g_{name}: {_rel(a, b):.2e}")
    assert bad == [], (bad, n_und)
    return mine, n_und


@pytest.mark.gpu
@pytest.mark.parametrize("B,N,D,K,S,form", [
    (3, 64 ** 3, 80, 2, 12, "centers"),          # LaRa's size
    (3, 64 ** 3, 80, 2, 12, "offset"),
    (1, 4097, 80, 2, 12, "centers"),             # rows not a multiple of the tile
    (1, 1, 80, 2, 12, "centers"),
    (1, 1, 80, 2, 12, "offset"),
    (1, 3001, 16, 1, 3, "centers"),
    (2, 1500, 48, 3, 27, "offset"),
    (1, 2000, 128, 4, 48, "centers"),            # weights read through L1
    (1, 2000, 128, 1, 12, "offset"),
    (1, 777, 112, 4, 27, "centers"),
    (1, 999, 32, 3, 48, "centers"),
    (1, 999, 64, 4, 3, "offset"),
    (1, 999, 96, 2, 27, "centers"),
])
def test_coarse_head_kernel_matches_float64(cuda_device, B, N, D, K, S, form):
    _accuracy_case(cuda_device, B, N, D, K, S, form)


@pytest.mark.gpu
def test_coarse_head_zero_rows_give_empty_outputs_and_zero_gradients(cuda_device):
    dev = cuda_device
    params = [p.to(dev) for p in random_params(80, 2, 12, 1)]
    head = _head(80, 2, 12, params, dev)
    feats = torch.zeros((1, 0, 80), device=dev, requires_grad=True)
    outs = head.forward_coarse(feats, OPACITY_SHIFT, SCALING_SHIFT)
    assert [tuple(o.shape) for o in outs] == [(1, 0, 3), (1, 0, 4, 3), (1, 0, 2), (1, 0, 4), (1, 0, 1)]
    sum(o.sum() for o in outs).backward()
    assert feats.grad.shape == feats.shape
    assert all(p.grad is not None and not bool(p.grad.any()) for p in head._params())


@pytest.mark.gpu
@pytest.mark.parametrize("logit", [30.0, -30.0])
def test_coarse_head_saturated_offsets(cuda_device, logit):
    _accuracy_case(cuda_device, 1, 4097, 80, 2, 12, "centers", seed=3, logit=logit)
    _accuracy_case(cuda_device, 1, 4097, 80, 2, 12, "offset", seed=3, logit=logit)


@pytest.mark.gpu
def test_coarse_head_mostly_dead_relus(cuda_device):
    _, n_und = _accuracy_case(cuda_device, 2, 20000, 80, 2, 12, "centers", seed=4, bias=-1.0)


@pytest.mark.gpu
def test_coarse_head_channels_last_feats(cuda_device):
    _accuracy_case(cuda_device, 2, 4097, 80, 2, 12, "centers", seed=5, strided=True)


def _bits(head, feats, gc, ups):
    outs, gx, gp = _run_kernel(head, feats, gc, ups, LARA_HALF_CELL)
    return outs + [gx] + [p.clone() for p in gp]


@pytest.mark.gpu
def test_coarse_head_is_bit_reproducible_with_the_deterministic_switch_off_and_on(cuda_device):
    dev = cuda_device
    g = torch.Generator().manual_seed(9)
    B, N, D, K, S = 3, 32 ** 3, 80, 2, 12
    params = [p.to(dev) for p in random_params(D, K, S, 9)]
    head = _head(D, K, S, params, dev)
    feats = torch.randn((B, N, D), generator=g).to(dev)
    gc = (torch.rand((N, 3), generator=g) - 0.5).to(dev)
    G = N * K
    ups = [torch.randn(s, generator=g).to(dev) for s in ((B, G, 3), (B, G, S // 3, 3), (B, G, 2), (B, G, 4),
                                                          (B, G, 1))]
    runs = []
    was = torch.are_deterministic_algorithms_enabled()
    try:
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            runs.append(_bits(head, feats, gc, ups))
            runs.append(_bits(head, feats, gc, ups))
    finally:
        torch.use_deterministic_algorithms(was)
    for r in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(runs[0], r))


@pytest.mark.gpu
def test_coarse_head_under_bf16_autocast_is_the_fp32_call(cuda_device):
    dev = cuda_device
    g = torch.Generator().manual_seed(12)
    B, N, D, K, S = 2, 5000, 80, 2, 12
    params = [p.to(dev) for p in random_params(D, K, S, 12)]
    head = _head(D, K, S, params, dev)
    feats = torch.randn((B, N, D), generator=g).to(dev).bfloat16()
    gc = (torch.rand((N, 3), generator=g) - 0.5).to(dev)
    with torch.no_grad():
        ref = head.gaussians(feats.float(), gc, OPACITY_SHIFT, SCALING_SHIFT, LARA_HALF_CELL)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            got = head.gaussians(feats, gc, OPACITY_SHIFT, SCALING_SHIFT, LARA_HALF_CELL)
    assert all(a.dtype == torch.float32 and torch.equal(a, b) for a, b in zip(got, ref))
    x = feats.clone().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        outs = head.gaussians(x, gc, OPACITY_SHIFT, SCALING_SHIFT, LARA_HALF_CELL)
    sum(o.float().sum() for o in outs).backward()
    assert x.grad.dtype == torch.bfloat16 and all(p.grad.dtype == torch.float32 for p in head._params())


@pytest.mark.gpu
def test_coarse_head_feeds_the_rasterizer_like_torchs_mlp_and_layout(cuda_device):
    """CoarseHead.gaussians -> render_scene_views(raw_activations=True) -> scene_loss -> backward matches the same chain
    through torch's mlp_coarse + gaussians_from_decoder to 1e-4 of each tensor's maximum.  The torch chain renders the
    head's values (its own enter the graph straight-through), so both chains share the rasterizer's discrete decisions
    (alpha and transmittance cut-offs), which fp32 differences of 1e-7 in a Gaussian can flip."""
    from lara_b200 import rasterizer as R
    from lara_b200 import scene as SC
    from lara_b200.decoder_layout import gaussians_from_decoder
    from lara_b200.loss import scene_loss
    from lara_b200.multiview import render_scene_views
    from oracle.coarse_head_torch import mlp_coarse_torch
    from test_point_feats import lara_cameras
    dev = cuda_device
    B, Rg, D, K, S, H, W, V = 1, 16, 80, 2, 12, 96, 96, 4
    N = Rg ** 3
    g = torch.Generator().manual_seed(13)
    params = random_params(D, K, S, 13)
    params[5] = params[5] + torch.tensor(([0.0] * 3 + [0.0] * S + [2.0] + [0.0] * 2 + [1.0, 0.0, 0.0, 0.0]) * K)
    params = [p.to(dev) for p in params]
    head = _head(D, K, S, params, dev)
    lin = (torch.arange(Rg, dtype=torch.float32) + 0.5) / Rg - 0.5
    gc = torch.stack(torch.meshgrid(lin, lin, lin, indexing="ij"), -1).reshape(N, 3).to(dev) * 0.5
    feats0 = torch.randn((B, N, D), generator=g).to(dev)
    cams, _, _ = lara_cameras(V, H, W, 5)
    settings = [SC.settings_for(c, torch.ones(3), 1, dev, R.GaussianRasterizationSettings) for c in cams]
    tar = torch.rand((V, H, W, 3), generator=g).to(dev)
    rays = torch.cat([torch.zeros(V, H, W, 3), torch.nn.functional.normalize(torch.randn((V, H, W, 3), generator=g),
                                                                             dim=-1)], -1).to(dev)
    half_cell = 0.5 * 0.5 / Rg
    grads = []
    for kind in ("kernel", "torch"):
        x = feats0.clone().requires_grad_(True)
        head.zero_grad(set_to_none=True)
        if kind == "kernel":
            gauss = head.gaussians(x, gc, OPACITY_SHIFT, SCALING_SHIFT, half_cell)
            values = [t.detach() for t in gauss]
        else:
            y = mlp_coarse_torch(x, head._params())
            gauss = [v + (t - t.detach()) for t, v in zip(
                gaussians_from_decoder(y, gc, K, S, OPACITY_SHIFT, SCALING_SHIFT, half_cell), values)]
        centers, shs, scaling, rotation, opacity = gauss
        out = render_scene_views(centers[0], shs[0], opacity[0], scaling[0], rotation[0], settings,
                                 rays=rays, raw_activations=True)
        loss, _ = scene_loss(out, tar, 2000)
        loss.backward()
        r = {"feats": x.grad.detach().clone()}
        r.update({k: p.grad.detach().clone() for k, p in head.named_parameters()})
        grads.append(r)
    bad = {k: _rel(grads[0][k], grads[1][k]) for k in grads[0]}
    assert {k: e for k, e in bad.items() if not e < 1e-4} == {}, bad


if __name__ == "__main__":
    # python tests/test_coarse_head.py OUT_DIR LARA_CHECKOUT: record LaRa's outputs, as
    # tests/golden/make_reference_records.py does for the other modules
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_reference_records import save
    out_dir, lara = sys.argv[1:3]
    os.makedirs(out_dir, exist_ok=True)
    save(out_dir, "test_coarse_head", record_reference(lara, "cpu"))
