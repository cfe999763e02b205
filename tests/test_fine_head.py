"""Fine-pass decoder head (Decoder.forward_fine, lightning/network.py:280-284, with the gathers and residual of
:508-512).

* CPU: the torch restatement ``oracle.fine_head_torch`` is pinned bit for bit against LaRa's own ``Decoder``
  (``norm`` + ``cross_att`` + ``mlp_fine``) with the mask gathers and residual around it: values, the three input
  gradients and the ten parameter gradients under a seeded upstream gradient.  LaRa's outputs are recorded in
  tests/golden/reference/test_fine_head.npz by record_reference:

      python tests/test_fine_head.py OUT_DIR LARA_CHECKOUT && cp OUT_DIR/test_fine_head.npz tests/golden/reference/

  ``FineHead``'s state-dict keys and shapes equal the recorded ones of LaRa's ``Decoder``; the argument checks of
  the Python entries and of the C entries run without a GPU.
* GPU: the kernels against the float64 restatement (every element of every output and gradient within 1e-5 of the
  tensor's maximum), the gather mode against LaRa's expression, bit-reproducibility with the deterministic switch off
  and on, and the fine pass end to end through the renderer and the loss.
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from helpers import fingerprint, reference_record
from test_decoder_layout import _import_reference_network

PARAM_NAMES = ("norm.weight", "norm.bias", "cross_att.q_proj_weight", "cross_att.k_proj_weight",
               "cross_att.v_proj_weight", "cross_att.out_proj.weight", "mlp_fine.0.weight", "mlp_fine.0.bias",
               "mlp_fine.2.weight", "mlp_fine.2.bias")
TOL = 1e-5


def random_params(D, S, seed, dtype=torch.float32):
    """The ten head parameters, seeded, at the scale of LaRa's initialisation, with non-trivial norm affine and
    biases."""
    g = torch.Generator().manual_seed(seed)

    def u(*shape, fan):
        return ((torch.rand(shape, generator=g) * 2 - 1) * (6.0 / fan) ** 0.5).to(dtype)
    return [1 + 0.2 * torch.randn(D, generator=g).to(dtype), 0.1 * torch.randn(D, generator=g).to(dtype),
            u(D, D, fan=2 * D), u(D, 8, fan=D + 8), u(D, 8, fan=D + 8), u(D, D, fan=2 * D),
            u(64, D, fan=D + 64), 0.1 * torch.randn(64, generator=g).to(dtype), u(S, 64, fan=64 + S),
            0.1 * torch.randn(S, generator=g).to(dtype)]


def state_signature(module_or_sd):
    sd = module_or_sd if isinstance(module_or_sd, dict) else module_or_sd.state_dict()
    return ";".join(f"{k}:{tuple(v.shape)}" for k, v in sorted(sd.items()))


# ---- CPU: restatement vs LaRa's own code ----------------------------------------------------------------------
N_CPU, K_CPU, D_CPU, V_CPU, S_CPU = 700, 2, 80, 4, 12


def _cpu_case():
    g = torch.Generator().manual_seed(21)
    vf = torch.randn((N_CPU, D_CPU), generator=g)
    mask = torch.rand(N_CPU * K_CPU, generator=g) < 0.7
    n = int(mask.sum())
    pf = torch.rand((V_CPU, 8, n), generator=g) * 2
    shs = torch.randn((N_CPU * K_CPU, S_CPU // 3, 3), generator=g)
    up = torch.randn((n, S_CPU // 3, 3), generator=g)
    return vf, mask, pf, shs, up


def _grads_record(out, leaves, params):
    rec = {"out": fingerprint(out.detach().numpy())}
    rec.update({"g_" + k: fingerprint(v.grad.numpy()) for k, v in leaves.items()})
    rec.update({"g_" + k: fingerprint(p.grad.numpy()) for k, p in zip(PARAM_NAMES, params)})
    return rec


def record_reference(lara, dev):
    """LaRa's own Decoder.forward_fine with the gathers and residual of network.py:508-512, on the CPU."""
    net = _import_reference_network(lara)
    dec = net.Decoder(D_CPU, S_CPU, 2, 4, 1, K=K_CPU)
    fine = {k: v for k, v in dec.state_dict().items() if not k.startswith("mlp_coarse")}
    sd = dict(zip(PARAM_NAMES, random_params(D_CPU, S_CPU, 5)))
    dec.load_state_dict(sd, strict=False)
    vf, mask, pf, shs, up = _cpu_case()
    leaves = {"volume_feat_up": vf.clone().requires_grad_(True), "point_feats": pf.clone().requires_grad_(True),
              "shs_coarse": shs.clone().requires_grad_(True)}
    point_feats = torch.einsum("lcb->blc", leaves["point_feats"])
    vpf = leaves["volume_feat_up"].unsqueeze(1).expand(-1, K_CPU, -1)[mask.view(-1, K_CPU)]
    out = dec.forward_fine(vpf, point_feats).view(-1, S_CPU // 3, 3) + leaves["shs_coarse"][mask]
    out.backward(up)
    params = [dict(dec.named_parameters())[k] for k in PARAM_NAMES]
    return {"fine_shs": _grads_record(out, leaves, params), "state": {"signature": np.array(state_signature(fine))}}


def test_fine_head_restatement_matches_reference_on_cpu():
    from oracle.fine_head_torch import fine_shs_torch
    vf, mask, pf, shs, up = _cpu_case()
    leaves = {"volume_feat_up": vf.clone().requires_grad_(True), "point_feats": pf.clone().requires_grad_(True),
              "shs_coarse": shs.clone().requires_grad_(True)}
    params = [p.requires_grad_(True) for p in random_params(D_CPU, S_CPU, 5)]
    out = fine_shs_torch(leaves["volume_feat_up"], K_CPU, mask, leaves["point_feats"], leaves["shs_coarse"], params)
    out.backward(up)
    mine = _grads_record(out, leaves, params)
    ref = reference_record("test_fine_head", "fine_shs")
    assert sorted(mine) == sorted(ref)
    assert [k for k in mine if mine[k] != ref[k]] == []


def test_fine_head_state_dict_matches_laras_decoder():
    from lara_b200.fine_head import FineHead
    head = FineHead(D_CPU, S_CPU)
    assert state_signature(head) == reference_record("test_fine_head", "state")["signature"]
    assert sorted(k for k, _ in head.named_parameters()) == sorted(PARAM_NAMES)


# ---- CPU: argument checks ----------------------------------------------------------------------------------------
def _small(n=5, V=2, D=16, S=12, N=4, K=2, dtype=torch.float32, dev="cpu"):
    g = torch.Generator().manual_seed(1)
    return (torch.randn((N, D), generator=g).to(dtype).to(dev), K,
            torch.tensor([True, False, True, True, False, True, True, False])[:N * K].to(dev),
            torch.randn((V, 8, n), generator=g).to(dtype).to(dev),
            torch.randn((N * K, S // 3, 3), generator=g).to(dtype).to(dev))


def test_fine_head_constructor_rejects_unsupported_sizes():
    from lara_b200.fine_head import FineHead
    for D, S in ((12, 12), (0, 12), (136, 12), (80, 9), (80, 75)):
        with pytest.raises(ValueError, match="FineHead"):
            FineHead(D, S)


@pytest.mark.parametrize("what", ["vf_dim", "mask_len", "mask_dtype", "shs", "pf_cond", "pf_views", "pf_count", "K"])
def test_fine_shs_rejects_bad_shapes(what):
    from lara_b200.fine_head import FineHead
    head = FineHead(16, 12)
    vf, K, mask, pf, shs = _small()
    bad = {"vf_dim": lambda: (vf[:, :8], K, mask, pf, shs),
           "mask_len": lambda: (vf, K, mask[:-1], pf, shs),
           "mask_dtype": lambda: (vf, K, mask.float(), pf, shs),
           "shs": lambda: (vf, K, mask, pf, shs[:, :1]),
           "pf_cond": lambda: (vf, K, mask, pf[:, :4], shs),
           "pf_views": lambda: (vf, K, mask, torch.zeros((9, 8, 5)), shs),
           "pf_count": lambda: (vf, K, mask, pf[:, :, :4], shs),
           "K": lambda: (vf, 0, mask, pf, shs)}[what]()
    with pytest.raises(RuntimeError, match="FineHead.fine_shs"):
        head.fine_shs(*bad)


def test_fine_head_rejects_dtype_and_device_before_any_launch():
    from lara_b200.fine_head import FineHead
    head = FineHead(16, 12)
    with pytest.raises(RuntimeError, match="Float"):
        head.fine_shs(*_small(dtype=torch.float64))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        head.fine_shs(*_small())
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        head.forward_fine(torch.zeros((5, 16)), torch.zeros((5, 3, 8)))
    with pytest.raises(RuntimeError, match="FineHead.forward_fine"):
        head.forward_fine(torch.zeros((5, 16)), torch.zeros((4, 3, 8)))
    with pytest.raises(RuntimeError, match="FineHead.forward_fine"):
        head.forward_fine(torch.zeros((5, 8)), torch.zeros((5, 3, 8)))
    with pytest.raises(RuntimeError, match="FineHead.forward_fine"):
        head.forward_fine(torch.zeros((5, 16)), torch.zeros((5, 9, 8)))


def test_fine_head_c_entries_reject_bad_sizes_before_any_launch(lib):
    P = ctypes.c_void_p(256)           # never dereferenced: the checks come before any CUDA call
    w = [P] * 10
    size = ctypes.c_size_t()
    bad = [(4, 2, 12, 12), (4, 2, 0, 12), (4, 2, 136, 12), (4, 0, 16, 12), (4, 9, 16, 12), (4, 2, 16, 9),
           (4, 2, 16, 75), (-1, 2, 16, 12)]
    for n, V, D, S in bad:
        assert lib.srf_fine_head_forward(None, n, V, D, S, 1, 4, P, None, P, None, *w, P) != 0
        assert b"srf_fine_head_forward: bad sizes" in lib.srf_last_error()
        assert lib.srf_fine_head_backward(None, n, V, D, S, 1, 4, P, None, P, *w, P, P, P, P, None, *w) != 0
        assert b"srf_fine_head_backward: bad sizes" in lib.srf_last_error()
        assert lib.srf_fine_head_workspace_bytes(n, V, D, S, 0, ctypes.byref(size)) != 0
        assert b"srf_fine_head_workspace_bytes: bad sizes" in lib.srf_last_error()
    # gather mode: K >= 1 and n <= N * K
    assert lib.srf_fine_head_forward(None, 4, 2, 16, 12, 0, 4, P, P, P, P, *w, P) != 0
    assert b"bad sizes" in lib.srf_last_error()
    assert lib.srf_fine_head_forward(None, 9, 2, 16, 12, 2, 4, P, P, P, P, *w, P) != 0
    assert b"bad sizes" in lib.srf_last_error()


def test_fine_head_c_entries_reject_null_pointers_before_any_launch(lib):
    P = ctypes.c_void_p(256)
    w = [P] * 10
    for k in range(10):
        nulled = list(w)
        nulled[k] = None
        assert lib.srf_fine_head_forward(None, 4, 2, 16, 12, 1, 4, P, None, P, None, *nulled, P) != 0
        assert b"null weight pointer" in lib.srf_last_error()
        assert lib.srf_fine_head_backward(None, 4, 2, 16, 12, 1, 4, P, None, P, *nulled, P, P, P, P, None, *w) != 0
        assert b"null weight pointer" in lib.srf_last_error()
        assert lib.srf_fine_head_backward(None, 4, 2, 16, 12, 1, 4, P, None, P, *w, P, P, P, P, None, *nulled) != 0
        assert b"null weight-gradient pointer" in lib.srf_last_error()
    assert lib.srf_fine_head_forward(None, 4, 2, 16, 12, 1, 4, None, None, P, None, *w, P) != 0
    assert b"null input pointer" in lib.srf_last_error()
    assert lib.srf_fine_head_forward(None, 4, 2, 16, 12, 1, 4, P, None, P, None, *w, None) != 0
    assert b"null output pointer" in lib.srf_last_error()
    # the residual is a gather-mode input
    assert lib.srf_fine_head_forward(None, 4, 2, 16, 12, 1, 4, P, None, P, P, *w, P) != 0
    assert b"needs idx" in lib.srf_last_error()
    # the workspace must be 256-byte aligned
    assert lib.srf_fine_head_backward(None, 4, 2, 16, 12, 1, 4, P, None, P, *w, P, ctypes.c_void_p(264), P, P,
                                      None, *w) != 0
    assert b"workspace must be 256-byte aligned" in lib.srf_last_error()
    assert lib.srf_fine_head_backward(None, 4, 2, 16, 12, 1, 4, P, None, P, *w, None, P, P, P, None, *w) != 0
    assert b"null upstream gradient" in lib.srf_last_error()
    # n == 0 in plain mode: nothing to read or write in the forward
    assert lib.srf_fine_head_forward(None, 0, 2, 16, 12, 1, 0, None, None, None, None, *w, None) == 0


# ---- GPU ----------------------------------------------------------------------------------------------------------
def _max_score(vf, pf, params):
    """Largest |attention score| of the float64 head (pf [V,8,n])."""
    ln_w, ln_b, wq, wk = (p.double() for p in params[:4])
    D = vf.shape[1]
    hd = D // 8
    x = torch.nn.functional.layer_norm(vf.double(), (D,), ln_w, ln_b, 1e-5)
    q = (x @ wq.T).view(-1, 8, hd)                              # [n,H,hd]
    k = torch.einsum("jcn,hdc->njhd", pf.double(), wk.view(8, hd, 8))   # [n,V,H,hd]
    return float((torch.einsum("nhd,njhd->nhj", q, k) / hd ** 0.5).abs().max())


def _head(D, S, seed, dev):
    from lara_b200.fine_head import FineHead
    head = FineHead(D, S).to(dev)
    with torch.no_grad():
        for p, v in zip(head._params(), random_params(D, S, seed)):
            p.copy_(v)
    return head


def _torch_run(vf, pf, params, g):
    """fine_head_torch forward + backward: (out, [g_vf, g_pf], [param grads])."""
    from oracle.fine_head_torch import fine_head_torch
    vf = vf.clone().requires_grad_(True)
    pf = pf.clone().requires_grad_(True)
    ps = [p.detach().clone().requires_grad_(True) for p in params]
    out = fine_head_torch(vf, pf.permute(2, 0, 1), ps)
    out.backward(g.view(out.shape))
    return out.detach().view(g.shape), [vf.grad, pf.grad], [p.grad for p in ps]


def _param_grads(head):
    """The ten parameter gradients in PARAM_NAMES order (at in_dim 8 the q/k/v ones are row blocks of in_proj)."""
    a = head.cross_att
    qkv = a.in_proj_weight.grad.chunk(3) if a._qkv_same_embed_dim else \
        (a.q_proj_weight.grad, a.k_proj_weight.grad, a.v_proj_weight.grad)
    return [head.norm.weight.grad, head.norm.bias.grad, *qkv, a.out_proj.weight.grad] + \
        [p.grad for p in (head.mlp_fine[0].weight, head.mlp_fine[0].bias, head.mlp_fine[2].weight, head.mlp_fine[2].bias)]


def _kernel_run(head, vf, pf, g):
    vf = vf.clone().requires_grad_(True)
    pf = pf.clone().requires_grad_(True)
    head.zero_grad(set_to_none=True)
    out = head.forward_fine(vf, pf.permute(2, 0, 1))
    out.backward(g.view(out.shape))
    return out.detach().view(g.shape), [vf.grad, pf.grad], _param_grads(head)


def _err(a, ref):
    a, ref = a.double(), ref.double()
    if ref.numel() == 0:
        return 0.0
    m = float(ref.abs().max())
    return float((a - ref).abs().max()) / (m if m > 0 else 1.0)


def _compare(mine, f32, f64, names):
    bad = []
    for name, a, b, c in zip(names, mine, f32, f64):
        assert a.shape == c.shape, name
        e, e32 = _err(a, c), _err(b, c)
        if not e <= TOL:
            bad.append(f"{name}: kernel {e:.2e} (fp32 torch restatement {e32:.2e})")
    assert bad == [], bad


def _accuracy_case(dev, V, n, D, S, score=None, seed=0):
    g = torch.Generator().manual_seed(seed + n)
    params = random_params(D, S, seed)
    vf = (torch.randn((n, D), generator=g) * 0.5 + 0.3).to(dev)
    pf = (torch.rand((V, 8, n), generator=g) * 2).to(dev)
    up = torch.randn((n, S), generator=g).to(dev)
    if score is not None and n > 0:
        pf = pf * (score / _max_score(vf, pf, [p.to(dev) for p in params]))
    head = _head(D, S, seed, dev)
    mine = _kernel_run(head, vf, pf, up)
    f32 = _torch_run(vf, pf, [p.to(dev) for p in params], up)
    f64 = _torch_run(vf.double(), pf.double(), [p.to(dev).double() for p in params], up.double())
    names = ["out", "g_volume_feat", "g_point_feats"] + ["g_" + k for k in PARAM_NAMES]
    _compare(*([r[0]] + r[1] + r[2] for r in (mine, f32, f64)), names)
    return vf, pf


@pytest.mark.gpu
@pytest.mark.parametrize("V,n,D,S", [(4, 262144, 80, 12), (2, 1000, 80, 12), (3, 4097, 80, 12), (1, 1, 128, 48),
                                     (4, 0, 128, 48), (8, 515, 8, 3), (5, 333, 40, 27)])
def test_fine_head_kernel_matches_float64(cuda_device, V, n, D, S):
    _accuracy_case(cuda_device, V, n, D, S)


@pytest.mark.gpu
def test_fine_head_scores_of_100_do_not_overflow(cuda_device):
    vf, pf = _accuracy_case(cuda_device, 4, 4097, 80, 12, score=100.0, seed=3)
    params = [p.to(cuda_device) for p in random_params(80, 12, 3)]
    assert 99.0 < _max_score(vf, pf, params) < 101.0


def _gather_case(N, K, V, D, S, seed, dev):
    """volume_feat_up, mask, point_feats, shs_coarse, upstream; the mask has voxels with 0, 1 and K masked Gaussians."""
    g = torch.Generator().manual_seed(seed)
    vf = torch.randn((N, D), generator=g)
    counts = torch.randint(0, K + 1, (N,), generator=g)
    counts[: min(N, 3)] = torch.tensor([0, 1, K])[: min(N, 3)]
    mask = torch.zeros((N, K), dtype=torch.bool)
    for r in range(N):
        mask[r, torch.randperm(K, generator=g)[: int(counts[r])]] = True
    mask = mask.view(-1)
    n = int(mask.sum())
    pf = torch.rand((V, 8, n), generator=g) * 2
    shs = torch.randn((N * K, S // 3, 3), generator=g)
    up = torch.randn((n, S // 3, 3), generator=g)
    return [t.to(dev) for t in (vf, mask, pf, shs, up)]


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 2, 3])
def test_fine_shs_matches_laras_gather_expression(cuda_device, K):
    from oracle.fine_head_torch import fine_shs_torch
    dev = cuda_device
    N, V, D, S = 3001, 4, 80, 12
    vf, mask, pf, shs, up = _gather_case(N, K, V, D, S, 40 + K, dev)
    head = _head(D, S, 7, dev)
    params = [dict(head.named_parameters())[k] for k in PARAM_NAMES]
    res = []
    for kind in ("kernel", "f32", "f64"):
        dt = torch.float64 if kind == "f64" else torch.float32
        leaves = [t.to(dt).clone().requires_grad_(True) for t in (vf, pf, shs)]
        ps = [p.detach().to(dt).clone().requires_grad_(True) for p in params]
        if kind == "kernel":
            head.zero_grad(set_to_none=True)
            out = head.fine_shs(leaves[0], K, mask, leaves[1], leaves[2])
            ps = params
        else:
            out = fine_shs_torch(leaves[0], K, mask, leaves[1], leaves[2], ps)
        out.backward(up.to(dt))
        res.append([out.detach()] + [t.grad for t in leaves] + [p.grad for p in ps])
    names = ["out", "g_volume_feat_up", "g_point_feats", "g_shs_coarse"] + ["g_" + k for k in PARAM_NAMES]
    _compare(res[0], res[1], res[2], names)
    empty = ~mask.view(N, K).any(1)
    assert bool(empty.any()) and not bool(res[0][1][empty].any())       # voxels without a masked Gaussian: exactly 0
    assert not bool(res[0][3][~mask].any())                             # unmasked residual rows: exactly 0
    assert torch.equal(res[0][3][mask], up)


def _bits(head, vf, mask, pf, shs, up, K):
    leaves = [t.clone().requires_grad_(True) for t in (vf, pf, shs)]
    head.zero_grad(set_to_none=True)
    out = head.fine_shs(leaves[0], K, mask, leaves[1], leaves[2])
    out.backward(up)
    return [out.detach()] + [t.grad for t in leaves] + [p.grad.clone() for p in head.parameters()]


@pytest.mark.gpu
def test_fine_head_is_bit_reproducible_with_the_deterministic_switch_off_and_on(cuda_device):
    dev = cuda_device
    vf, mask, pf, shs, up = _gather_case(131072, 2, 4, 80, 12, 9, dev)
    head = _head(80, 12, 9, dev)
    runs = []
    was = torch.are_deterministic_algorithms_enabled()
    try:
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            runs.append(_bits(head, vf, mask, pf, shs, up, 2))
            runs.append(_bits(head, vf, mask, pf, shs, up, 2))
    finally:
        torch.use_deterministic_algorithms(was)
    for r in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(runs[0], r))


@pytest.mark.gpu
def test_fine_pass_end_to_end_through_renderer_and_loss(cuda_device):
    """render_scene_views (coarse) -> sample_point_feats -> fine_shs -> render_scene_views on the masked Gaussians ->
    scene_loss(prex="_fine") -> backward: the Gaussian-parameter, voxel-feature and head-weight gradients match the same
    chain through the fp32 restatement."""
    from lara_b200 import rasterizer as R
    from lara_b200 import scene as S
    from lara_b200.loss import scene_loss
    from lara_b200.multiview import render_scene_views
    from lara_b200.point_feats import sample_point_feats
    from oracle.fine_head_torch import fine_shs_torch
    from test_point_feats import lara_cameras
    dev = cuda_device
    K, H, W, V, n_sel, D, SH = 2, 96, 96, 4, 3, 80, 12
    sc = S.scene(6000, 3)
    P = sc["means3D"].shape[0]
    N = P // K
    cams, w2c, ixt = lara_cameras(V, H, W, 5)
    settings = [S.settings_for(c, torch.ones(3), sc["sh_degree"], dev, R.GaussianRasterizationSettings) for c in cams]
    g = torch.Generator().manual_seed(8)
    rays = torch.cat([torch.zeros(V, H, W, 3), torch.nn.functional.normalize(torch.randn((V, H, W, 3), generator=g),
                                                                             dim=-1)], -1).to(dev)
    img_ref = torch.rand((n_sel, 3, H, W), generator=g).to(dev)
    tar = torch.rand((V, H, W, 3), generator=g).to(dev)
    mask = (torch.rand(N * K, generator=g) < 0.6).to(dev)
    vf0 = torch.randn((N, D), generator=g).to(dev)
    head = _head(D, SH, 11, dev)
    grads = []
    for kind in ("kernel", "torch"):
        leaves = {k: sc[k][: N * K].to(dev).clone().requires_grad_(True)
                  for k in ("means3D", "shs", "opacities", "scales", "rotations")}
        vf = vf0.clone().requires_grad_(True)
        head.zero_grad(set_to_none=True)
        out = render_scene_views(leaves["means3D"], leaves["shs"], leaves["opacities"], leaves["scales"],
                                 leaves["rotations"], settings, rays=rays)
        rend = {k: out[k][:n_sel] for k in ("image", "acc_map", "depth")}
        pf = sample_point_feats(leaves["means3D"][mask], img_ref, rend, w2c[:n_sel].to(dev), ixt[:n_sel].to(dev))
        if kind == "kernel":
            shs_fine = head.fine_shs(vf, K, mask, pf, leaves["shs"])
        else:
            shs_fine = fine_shs_torch(vf, K, mask, pf, leaves["shs"], [dict(head.named_parameters())[k]
                                                                         for k in PARAM_NAMES])
        fine = render_scene_views(leaves["means3D"][mask], shs_fine, leaves["opacities"][mask],
                                  leaves["scales"][mask], leaves["rotations"][mask], settings, rays=rays, prex="_fine")
        loss, _ = scene_loss(out, tar, 2000)
        loss_fine, _ = scene_loss(fine, tar, 2000, prex="_fine")
        (loss + loss_fine).backward()
        r = {k: v.grad.detach().clone() for k, v in leaves.items()}
        r["volume_feat_up"] = vf.grad.detach().clone()
        r.update({k: p.grad.detach().clone() for k, p in head.named_parameters()})
        grads.append(r)
    bad = {k: _err(grads[0][k], grads[1][k]) for k in grads[0]}
    assert {k: e for k, e in bad.items() if not e < 1e-4} == {}, bad


if __name__ == "__main__":
    # python tests/test_fine_head.py OUT_DIR LARA_CHECKOUT: record LaRa's outputs, as tests/golden/make_reference_records.py
    # does for the other modules
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_reference_records import save
    out_dir, lara = sys.argv[1:3]
    os.makedirs(out_dir, exist_ok=True)
    save(out_dir, "test_fine_head", record_reference(lara, "cpu"))
