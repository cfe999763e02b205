"""Feature-volume lifting of LaRa's coarse pass (Network.build_feat_vol, lightning/network.py:352-379, the view-embedding
concatenation of :451-452 and VolTransformer.forward's blocks, :145-150).

* CPU: the torch restatement ``oracle.feat_volume_torch`` is pinned bit for bit against LaRa's own code -- ``ModLN``,
  ``projection``, ``rsh_cart_3``, ``ray_to_plucker`` and ``Network.build_feat_vol`` called on a stand-in ``self``,
  plus the condition ``VolTransformer.forward`` hands its first layer (captured with a forward pre-hook): values and
  the gradients of img_feats, the four ``dir_norm`` tensors and ``view_embed`` under a seeded upstream gradient.
  LaRa's outputs are recorded in tests/golden/reference/test_feat_volume.npz by record_reference:

      python tests/test_feat_volume.py OUT_DIR LARA_CHECKOUT && cp OUT_DIR/test_feat_volume.npz tests/golden/reference/

  ``FeatVolume``'s state-dict keys and shapes (and its voxel grid, bit for bit) equal the recorded ones of LaRa's
  ``Network``; the argument checks of the Python entries and of the C entries run without a GPU.
* GPU: bit-reproducibility with the deterministic switch off and on, and bf16 autocast.  Both layouts and every
  gradient are checked element by element against float64, the two layouts' bits against each other and a voxel slice
  in a camera's plane, in tests/test_feat_volume_per_element.py.
"""
import ctypes
import math
import os
import sys
import types

import numpy as np
import pytest
import torch

from helpers import fingerprint, reference_record
from test_decoder_layout import _import_reference_network

PARAM_NAMES = ("dir_norm.norm.weight", "dir_norm.norm.bias", "dir_norm.mlp.1.weight", "dir_norm.mlp.1.bias")
VMAX = 4


def cameras(B, V, H, W, seed, straddle=False, fov=0.8):
    """w2c [B,V,4,4] and ixt [B,V,3,3] (row-major, OpenCV axes) of cameras around the origin looking at it, and their
    centres [B,V,3].  With straddle, every odd view's principal point is moved so that the volume's projection
    crosses the image border."""
    g = torch.Generator().manual_seed(seed)
    w2c = torch.zeros(B, V, 4, 4, dtype=torch.float64)
    ixt = torch.zeros(B, V, 3, 3, dtype=torch.float64)
    centre = torch.zeros(B, V, 3, dtype=torch.float64)
    for b in range(B):
        for v in range(V):
            d = torch.randn(3, generator=g, dtype=torch.float64)
            c = d / d.norm() * (1.8 + 0.4 * float(torch.rand(1, generator=g)))
            fwd = -c / c.norm()
            up = torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64)
            right = torch.linalg.cross(fwd, up)
            right = right / right.norm()
            down = torch.linalg.cross(fwd, right)
            rot = torch.stack([right, down, fwd])
            w2c[b, v, :3, :3] = rot
            w2c[b, v, :3, 3] = -rot @ c
            w2c[b, v, 3, 3] = 1.0
            f = 0.5 * W / math.tan(0.5 * fov)
            cx, cy = W / 2, H / 2
            if straddle and v % 2 == 1:
                cx, cy = cx + 0.45 * W, cy - 0.3 * H
            ixt[b, v] = torch.tensor([[f, 0, cx], [0, f, cy], [0, 0, 1]], dtype=torch.float64)
            centre[b, v] = c
    return w2c.float(), ixt.float(), centre.float()


def make_case(B, V, C, h, w, H, W, R, E, seed, straddle=False):
    """Seeded inputs (CPU, fp32): img_feats, rays_down, w2cs, ixts, the four dir_norm tensors, view_embed or None."""
    g = torch.Generator().manual_seed(seed)
    w2c, ixt, centre = cameras(B, V, H, W, seed, straddle)
    img_feats = torch.randn((B * V, C, h, w), generator=g) * 1.5 + 0.4
    dirs = torch.randn((B, V, h, w, 3), generator=g)
    rays = torch.cat([centre[:, :, None, None].expand(B, V, h, w, 3) + 0.05 * torch.randn((B, V, h, w, 3), generator=g),
                      dirs], -1)
    params = [1 + 0.2 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g),
              (torch.rand((2 * C, 32), generator=g) * 2 - 1) / 32 ** 0.5, 0.1 * torch.randn(2 * C, generator=g)]
    ve = torch.randn((1, VMAX, E, 1, 1, 1), generator=g) / E ** 0.5 if E > 0 else None
    return img_feats, rays.contiguous(), w2c, ixt, params, ve


def torch_path(img_feats, rays, w2c, ixt, image_hw, grid, params, ve, n_group):
    """The restatement: build_feat_vol, then (n_group > 0) the view-embedding cat and the blocks."""
    from oracle.feat_volume_torch import build_feat_vol_torch, cond_tokens_torch
    vol = build_feat_vol_torch(img_feats, rays, w2c, ixt, image_hw, grid, params)
    return vol if n_group == 0 else cond_tokens_torch(vol, ve, n_group)


def state_signature(sd):
    return ";".join(f"{k}:{tuple(v.shape)}" for k, v in sorted(sd.items()))


# ---- CPU: restatement vs LaRa's own code ----------------------------------------------------------------------
CPU = dict(B=2, V=3, C=64, h=6, w=8, H=96, W=128, R=4)
CPU_CASES = {"dropin": (0, 0, False), "cond_g4": (4, 8, False), "cond_g2": (2, 8, False), "cond_g2_e0": (2, 0, False),
             "straddle_g2": (2, 8, True)}


def _cpu_inputs(name):
    n_group, E, straddle = CPU_CASES[name]
    c = CPU
    case = make_case(c["B"], c["V"], c["C"], c["h"], c["w"], c["H"], c["W"], c["R"], E, 31 + len(name), straddle)
    shape = (c["B"], c["V"], c["C"], c["R"], c["R"], c["R"]) if n_group == 0 else \
        (c["B"] * n_group ** 3, c["V"] * (c["R"] // n_group) ** 3, c["C"] + E)
    up = torch.randn(shape, generator=torch.Generator().manual_seed(7))
    return case, n_group, up


def _record(out, img_feats, params, ve):
    rec = {"out": fingerprint(out.detach().numpy()), "g_img_feats": fingerprint(img_feats.grad.numpy())}
    rec.update({"g_" + k: fingerprint(p.grad.numpy()) for k, p in zip(PARAM_NAMES, params)})
    if ve is not None:
        rec["g_view_embed"] = fingerprint(ve.grad.numpy())
    return rec


class _Captured(Exception):
    pass


def _lara_case(net, name):
    (img_feats, rays, w2c, ixt, params, ve), n_group, up = _cpu_inputs(name)
    c = CPU
    B, V, R = c["B"], c["V"], c["R"]
    dir_norm = net.ModLN(c["C"], 16 * 2, eps=1e-6)
    dir_norm.load_state_dict({"norm.weight": params[0], "norm.bias": params[1], "mlp.1.weight": params[2],
                              "mlp.1.bias": params[3]})
    fake = types.SimpleNamespace(device=torch.device("cpu"), scene_size=0.5, feat_vol_reso=R, dir_norm=dir_norm)
    fake.volume_grid = net.Network.build_dense_grid(fake, R)
    fake.ray_to_plucker = lambda r: net.Network.ray_to_plucker(fake, r)
    x = img_feats.clone().requires_grad_(True)
    batch = {"tar_ixt": ixt, "tar_w2c": w2c, "tar_rays_down": rays}
    src_inps = torch.zeros((B * V, 3, c["H"], c["W"]))
    out = net.Network.build_feat_vol(fake, src_inps, x, V, batch)
    view_embed = torch.nn.Parameter(ve.clone()) if ve is not None else None
    if n_group > 0:
        feat_vol = out
        if view_embed is not None:       # network.py:451-452
            feat_vol = torch.cat((feat_vol, view_embed[:, :V].expand(B, -1, -1, R, R, R)), dim=2)
        vt = net.VolTransformer(embed_dim=8, image_feat_dim=feat_vol.shape[2], n_groups=[n_group], vol_low_res=R,
                                vol_high_res=2 * R, out_dim=4, num_layers=1, num_heads=1)
        seen = []

        def hook(module, args):
            seen.append(args[1])
            raise _Captured()
        vt.layers[0].register_forward_pre_hook(hook)
        try:
            vt(feat_vol)
        except _Captured:
            pass
        out = seen[0]
    out.backward(up)
    return _record(out, x, [dir_norm.norm.weight, dir_norm.norm.bias, dir_norm.mlp[1].weight, dir_norm.mlp[1].bias],
                   view_embed), fake.volume_grid


def record_reference(lara, dev):
    """LaRa's own build_feat_vol, view-embedding cat and VolTransformer blocks on the CPU."""
    net = _import_reference_network(lara)
    recs = {}
    for name in CPU_CASES:
        recs[name], grid = _lara_case(net, name)
    E = 8
    sd = {"dir_norm." + k: v for k, v in net.ModLN(CPU["C"], 16 * 2, eps=1e-6).state_dict().items()}
    sd["view_embed"] = torch.zeros(1, 4, E, 1, 1, 1)      # network.py:310
    sd["volume_grid"] = grid
    recs["state"] = {"signature": np.array(state_signature(sd)), "volume_grid": fingerprint(grid.numpy())}
    return recs


@pytest.mark.parametrize("name", sorted(CPU_CASES))
def test_feat_volume_restatement_matches_reference_on_cpu(name):
    from lara_b200.feat_volume import dense_grid
    (img_feats, rays, w2c, ixt, params, ve), n_group, up = _cpu_inputs(name)
    x = img_feats.clone().requires_grad_(True)
    ps = [p.clone().requires_grad_(True) for p in params]
    v = ve.clone().requires_grad_(True) if ve is not None else None
    out = torch_path(x, rays, w2c, ixt, (CPU["H"], CPU["W"]), dense_grid(CPU["R"]), ps, v, n_group)
    out.backward(up)
    mine = _record(out, x, ps, v)
    ref = reference_record("test_feat_volume", name)
    assert sorted(mine) == sorted(ref)
    assert [k for k in mine if mine[k] != ref[k]] == []


def test_feat_volume_state_dict_matches_laras_network():
    from lara_b200.feat_volume import FeatVolume
    fv = FeatVolume(CPU["C"], 8, CPU["R"])
    ref = reference_record("test_feat_volume", "state")
    assert state_signature(fv.state_dict()) == ref["signature"]
    assert fingerprint(fv.volume_grid.numpy()) == ref["volume_grid"]
    assert sorted(k for k, _ in fv.named_parameters()) == sorted(PARAM_NAMES + ("view_embed",))


# ---- CPU: argument checks ----------------------------------------------------------------------------------------
def _small(B=1, V=2, C=32, h=3, w=4, dev="cpu", dtype=torch.float32):
    g = torch.Generator().manual_seed(2)
    return (torch.randn((B * V, C, h, w), generator=g).to(dtype).to(dev),
            torch.randn((B, V, h, w, 6), generator=g).to(dtype).to(dev),
            torch.eye(4).expand(B, V, 4, 4).to(dtype).to(dev), torch.eye(3).expand(B, V, 3, 3).to(dtype).to(dev),
            (48, 64))


def test_feat_volume_constructor_rejects_unsupported_sizes():
    from lara_b200.feat_volume import FeatVolume
    for C, E, R in ((48, 8, 4), (0, 8, 4), (1056, 8, 4), (32, -1, 4), (32, 129, 4), (32, 8, 0), (32, 8, 65)):
        with pytest.raises(ValueError, match="FeatVolume"):
            FeatVolume(C, E, R)


@pytest.mark.parametrize("what", ["rays_rank", "rays_last", "views", "img_feats", "w2cs", "ixts", "image_hw",
                                  "n_group", "too_many_views"])
def test_feat_volume_rejects_bad_shapes(what):
    from lara_b200.feat_volume import FeatVolume
    fv = FeatVolume(32, 8, 4)
    x, rays, w2c, ixt, hw = _small()
    args = {"rays_rank": lambda: (x, rays[0], w2c, ixt, hw, 2),
            "rays_last": lambda: (x, rays[..., :5], w2c, ixt, hw, 2),
            "views": lambda: (torch.zeros((9, 32, 3, 4)), torch.zeros((1, 9, 3, 4, 6)), w2c, ixt, hw, 2),
            "img_feats": lambda: (x[:, :16], rays, w2c, ixt, hw, 2),
            "w2cs": lambda: (x, rays, w2c[..., :3, :], ixt, hw, 2),
            "ixts": lambda: (x, rays, w2c, ixt[:, :1], hw, 2),
            "image_hw": lambda: (x, rays, w2c, ixt, (0, 64), 2),
            "n_group": lambda: (x, rays, w2c, ixt, hw, 3),
            "too_many_views": lambda: (torch.zeros((5, 32, 3, 4)), torch.zeros((1, 5, 3, 4, 6)),
                                       torch.zeros((1, 5, 4, 4)), torch.zeros((1, 5, 3, 3)), hw, 2)}[what]()
    with pytest.raises(RuntimeError, match="FeatVolume.cond_tokens"):
        fv.cond_tokens(*args)


def test_feat_volume_rejects_dtype_device_and_constant_grads_before_any_launch():
    from lara_b200.feat_volume import FeatVolume
    fv = FeatVolume(32, 8, 4)
    with pytest.raises(RuntimeError, match="Float"):
        fv(*_small(dtype=torch.float64))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        fv(*_small())
    x, rays, w2c, ixt, hw = _small()
    for i, name in ((1, "rays_down"), (2, "w2cs"), (3, "ixts")):
        args = [x, rays, w2c, ixt, hw]
        args[i] = args[i].clone().requires_grad_(True)
        with pytest.raises(RuntimeError, match=f"{name} requires grad"):
            fv.cond_tokens(*args, 2)
    fv.dir_norm.norm.weight.data = torch.zeros(16)
    with pytest.raises(RuntimeError, match="dir_norm.norm.weight must be"):
        fv(x, rays, w2c, ixt, hw)


def _c_args(B=1, V=2, C=32, h=3, w=4, R=4, E=8, Vmax=4, H=48, W=64, ng=2):
    return [B, V, C, h, w, R, E, Vmax, H, W, ng]


def test_feat_volume_c_entries_reject_bad_sizes_before_any_launch(lib):
    P = ctypes.c_void_p(256)           # never dereferenced: the checks come before any CUDA call
    size = ctypes.c_size_t()
    bad = [dict(B=0), dict(V=0), dict(V=9), dict(C=48), dict(C=0), dict(C=1056), dict(h=0), dict(w=0), dict(R=0),
           dict(R=65), dict(E=-1), dict(E=129)]
    for kw in bad:
        a = _c_args(**kw)
        assert lib.srf_feat_volume_forward(None, *a, P, P, P, P, P, P, P, P, P, P, P, P) != 0
        assert b"srf_feat_volume_forward: bad sizes" in lib.srf_last_error()
        assert lib.srf_feat_volume_backward(None, *a, P, P, P, P, P, P, P, P, P, P, P, P, P, P, P, P, P) != 0
        assert b"srf_feat_volume_backward: bad sizes" in lib.srf_last_error()
        assert lib.srf_feat_volume_workspace_bytes(*a[:7], ctypes.byref(size)) != 0
        assert b"srf_feat_volume_workspace_bytes: bad sizes" in lib.srf_last_error()
    for kw, msg in ((dict(Vmax=1), b"bad sizes (Vmax"), (dict(H=0), b"bad sizes (H_img"), (dict(W=0), b"bad sizes (H_img"),
                    (dict(ng=3), b"bad layout"), (dict(ng=-1), b"bad layout"), (dict(ng=0), b"bad layout")):
        assert lib.srf_feat_volume_forward(None, *_c_args(**kw), P, P, P, P, P, P, P, P, P, P, P, P) != 0
        assert msg in lib.srf_last_error()
    assert lib.srf_feat_volume_workspace_bytes(*_c_args()[:7], None) != 0
    assert lib.srf_feat_volume_workspace_bytes(*_c_args()[:7], ctypes.byref(size)) == 0 and size.value > 0


def test_feat_volume_c_entries_reject_null_pointers_before_any_launch(lib):
    P = ctypes.c_void_p(256)
    a = _c_args()
    msgs = [b"null input pointer"] * 5 + [b"null weight pointer"] * 4 + [b"null view_embed"]
    for k, msg in enumerate(msgs):
        ptrs = [P] * 12
        ptrs[k] = None
        assert lib.srf_feat_volume_forward(None, *a, *ptrs) != 0
        assert msg in lib.srf_last_error()
    assert lib.srf_feat_volume_forward(None, *a, *([P] * 11), None) != 0
    assert b"null output pointer" in lib.srf_last_error()
    assert lib.srf_feat_volume_forward(None, *a, *([P] * 10), ctypes.c_void_p(264), P) != 0
    assert b"workspace must be 256-byte aligned" in lib.srf_last_error()
    msgs = [b"null input pointer"] * 5 + [b"null weight pointer"] * 4 + [b"null upstream gradient"] + \
        [b"workspace must be"] + [b"null gradient pointer"] * 6
    for k, msg in enumerate(msgs):
        ptrs = [P] * 17
        ptrs[k] = None
        assert lib.srf_feat_volume_backward(None, *a, *ptrs) != 0
        assert msg in lib.srf_last_error()
    # E = 0 needs no view_embed and no d_view_embed
    a0 = _c_args(E=0)
    assert lib.srf_feat_volume_backward(None, *a0, *([P] * 10), ctypes.c_void_p(264), *([P] * 5), None) != 0
    assert b"workspace must be 256-byte aligned" in lib.srf_last_error()


# ---- GPU ----------------------------------------------------------------------------------------------------------
def _module(case, C, E, R, dev):
    from lara_b200.feat_volume import FeatVolume
    _, _, _, _, params, ve = case
    fv = FeatVolume(C, E, R).to(dev)
    with torch.no_grad():
        for p, v in zip((fv.dir_norm.norm.weight, fv.dir_norm.norm.bias, fv.dir_norm.mlp[1].weight,
                         fv.dir_norm.mlp[1].bias), params):
            p.copy_(v)
        if E > 0:
            fv.view_embed.copy_(ve)
    return fv


def _grads(fv):
    gs = [fv.dir_norm.norm.weight.grad, fv.dir_norm.norm.bias.grad, fv.dir_norm.mlp[1].weight.grad,
          fv.dir_norm.mlp[1].bias.grad]
    return gs + ([fv.view_embed.grad] if fv.view_embed_dim > 0 else [])


def _kernel_run(fv, case, image_hw, n_group, up, dev):
    x = case[0].to(dev).requires_grad_(True)
    args = [t.to(dev) for t in case[1:4]]
    fv.zero_grad(set_to_none=True)
    out = fv(x, *args, image_hw) if n_group == 0 else fv.cond_tokens(x, *args, image_hw, n_group)
    out.backward(up)
    return [out.detach(), x.grad] + [g.clone() for g in _grads(fv)[: 4 + (n_group > 0 and fv.view_embed_dim > 0)]]


# B, V, C, (h, w), (H_img, W_img), R, E, n_group, straddle
GPU_CASES = {
    "lara": (3, 4, 768, (32, 32), (512, 512), 16, 32, 16, False),
    "c384": (3, 4, 384, (32, 32), (512, 512), 16, 32, 8, False),
}


def _bits(fv, case, hw, ng, up, dev):
    return _kernel_run(fv, case, hw, ng, up, dev)


@pytest.mark.gpu
def test_feat_volume_is_bit_reproducible_with_the_deterministic_switch_off_and_on(cuda_device):
    dev = cuda_device
    B, V, C, (h, w), hw, R, E, ng, _ = GPU_CASES["lara"]
    case = make_case(B, V, C, h, w, hw[0], hw[1], R, E, 11)
    fv = _module(case, C, E, R, dev)
    up = torch.randn((B * ng ** 3, V * (R // ng) ** 3, C + E), generator=torch.Generator().manual_seed(9)).to(dev)
    runs = []
    was = torch.are_deterministic_algorithms_enabled()
    try:
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            runs.append(_bits(fv, case, hw, ng, up, dev))
            runs.append(_bits(fv, case, hw, ng, up, dev))
    finally:
        torch.use_deterministic_algorithms(was)
    for r in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(runs[0], r))


@pytest.mark.gpu
def test_feat_volume_under_bf16_autocast_computes_in_fp32(cuda_device):
    dev = cuda_device
    B, V, C, (h, w), hw, R, E, ng, _ = GPU_CASES["c384"]
    case = make_case(B, V, C, h, w, hw[0], hw[1], R, E, 12)
    fv = _module(case, C, E, R, dev)
    args = [t.to(dev) for t in case[:4]]
    ref = fv.cond_tokens(*args, hw, ng)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = fv.cond_tokens(*args, hw, ng)
        bf = fv.cond_tokens(args[0].bfloat16(), *args[1:], hw, ng)
    assert out.dtype == torch.float32 and torch.equal(out, ref)
    assert bf.dtype == torch.float32 and torch.equal(bf, fv.cond_tokens(args[0].bfloat16().float(), *args[1:], hw, ng))


if __name__ == "__main__":
    # python tests/test_feat_volume.py OUT_DIR LARA_CHECKOUT: record LaRa's outputs, as tests/golden/make_reference_records.py
    # does for the other modules
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_reference_records import save
    out_dir, lara = sys.argv[1:3]
    os.makedirs(out_dir, exist_ok=True)
    save(out_dir, "test_feat_volume", record_reference(lara, "cpu"))
