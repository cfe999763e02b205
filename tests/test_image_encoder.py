"""LaRa's image encoder (DinoWrapper, lightning/network.py:14-55, 442-445): timm's DINO ViT with the patch and position
embedding and the residual LayerNorms in CUDA (lara_b200.image_encoder, csrc/image_encoder.cu).

* CPU: the restatement ``oracle.vit_torch`` against torchvision's ``vision_transformer.Encoder`` in float64 (weights
  mapped, the resampled ``pos_embed`` as its ``pos_embedding``) at 224^2 and 512^2 for both widths, on two blocks (the
  blocks are identical, so two pin the hand-off between them); the resample map against ``F.interpolate`` in float64;
  the patch matrix against ``transforms.Normalize`` + ``F.conv2d``; timm's state-dict keys and shapes, a LaRa checkpoint
  loaded strictly, and the argument checks of the Python and C entries.  With timm importable, the restatement against
  ``timm.create_model``; otherwise that test skips.
* GPU (TF32 off for the fp32 comparisons): the patch, token and final-norm kernels, forward and backward, against
  float64 (every element within 1e-5 of the tensor's float64 maximum); the residual LayerNorm (``srf_vit_layernorm``)
  element by element against a float64 statement with a bound per element, in
  tests/test_vol_transformer_per_element.py; the whole encoder's output and its 150 parameter gradients against float64,
  beside the fp32 restatement; bit-reproducibility under ``torch.use_deterministic_algorithms(True)`` and the same bits
  under ``no_grad``; the chain to ``FeatVolume`` through LaRa's einsum / reshape.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

TOL = 1e-5
WIDTHS = {768: 12, 384: 6}               # C -> heads
NAMES = {768: "vit_base_patch16_224.dino", 384: "vit_small_patch16_224.dino"}


def timm_keys(C, depth=12):
    """timm's ``VisionTransformer`` state dict for the DINO models: (name, shape) in its order."""
    keys = [("cls_token", (1, 1, C)), ("pos_embed", (1, 197, C)), ("patch_embed.proj.weight", (C, 3, 16, 16)),
            ("patch_embed.proj.bias", (C,))]
    for i in range(depth):
        b = f"blocks.{i}."
        keys += [(b + "norm1.weight", (C,)), (b + "norm1.bias", (C,)), (b + "attn.qkv.weight", (3 * C, C)),
                 (b + "attn.qkv.bias", (3 * C,)), (b + "attn.proj.weight", (C, C)), (b + "attn.proj.bias", (C,)),
                 (b + "norm2.weight", (C,)), (b + "norm2.bias", (C,)), (b + "mlp.fc1.weight", (4 * C, C)),
                 (b + "mlp.fc1.bias", (4 * C,)), (b + "mlp.fc2.weight", (C, 4 * C)), (b + "mlp.fc2.bias", (C,))]
    return keys + [("norm.weight", (C,)), ("norm.bias", (C,))]


def vit_params(C, depth, seed):
    """Seeded parameters under timm's names (fp32, CPU)."""
    g = torch.Generator().manual_seed(seed)
    p = {}
    for k, shape in timm_keys(C, depth):
        if k.endswith("norm1.weight") or k.endswith("norm2.weight") or k == "norm.weight":
            p[k] = 1 + 0.2 * torch.randn(shape, generator=g)
        elif k.endswith(".bias"):
            p[k] = 0.1 * torch.randn(shape, generator=g)
        elif k in ("cls_token", "pos_embed"):
            p[k] = 0.5 * torch.randn(shape, generator=g)
        else:
            fan = shape[1] if len(shape) == 2 else 3 * 16 * 16
            p[k] = (torch.rand(shape, generator=g) * 2 - 1) / fan ** 0.5
    return p


def images(N, H, W, seed):
    return torch.rand((N, 3, H, W), generator=torch.Generator().manual_seed(seed))


# ---- CPU: the restatement ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", sorted(WIDTHS))
@pytest.mark.parametrize("size", [224, 512])
def test_restatement_matches_torchvision_encoder_in_float64(C, size):
    from torchvision.models.vision_transformer import Encoder
    from oracle.vit_torch import patch_tokens, resample_pos_embed, vit_forward
    heads, depth = WIDTHS[C], 2
    p = {k: v.double() for k, v in vit_params(C, depth, 7 + size).items()}
    img = images(1, size, size, size).double()
    with torch.no_grad():
        mine = vit_forward(img, p, heads)
        enc = Encoder(seq_length=1 + (size // 16) ** 2, num_layers=depth, num_heads=heads, hidden_dim=C, mlp_dim=4 * C,
                      dropout=0.0, attention_dropout=0.0).double().eval()
        sd = {"pos_embedding": resample_pos_embed(p["pos_embed"], size // 16, size // 16), "ln.weight": p["norm.weight"],
              "ln.bias": p["norm.bias"]}
        for i in range(depth):
            b, e = f"blocks.{i}.", f"layers.encoder_layer_{i}."
            sd.update({e + "ln_1.weight": p[b + "norm1.weight"], e + "ln_1.bias": p[b + "norm1.bias"],
                       e + "self_attention.in_proj_weight": p[b + "attn.qkv.weight"],
                       e + "self_attention.in_proj_bias": p[b + "attn.qkv.bias"],
                       e + "self_attention.out_proj.weight": p[b + "attn.proj.weight"],
                       e + "self_attention.out_proj.bias": p[b + "attn.proj.bias"],
                       e + "ln_2.weight": p[b + "norm2.weight"], e + "ln_2.bias": p[b + "norm2.bias"],
                       e + "mlp.0.weight": p[b + "mlp.fc1.weight"], e + "mlp.0.bias": p[b + "mlp.fc1.bias"],
                       e + "mlp.3.weight": p[b + "mlp.fc2.weight"], e + "mlp.3.bias": p[b + "mlp.fc2.bias"]})
        enc.load_state_dict(sd, strict=True)
        # torchvision's Encoder adds pos_embedding itself: hand it the tokens without their position rows
        p0 = dict(p, pos_embed=torch.zeros_like(p["pos_embed"]))
        ref = enc(patch_tokens(img, p0))[:, 1:]
    assert float((mine - ref).abs().max()) <= 1e-12 * float(ref.abs().max())


@pytest.mark.parametrize("size", [(32, 32), (32, 24), (8, 8), (14, 14)])
def test_resample_map_matches_interpolate_in_float64(size):
    from lara_b200.image_encoder import resample_map
    h, w = size
    M = resample_map(h, w)
    assert M.dtype == torch.float64 and M.shape == (h * w, 196)
    if size == (14, 14):
        assert torch.equal(M, torch.eye(196, dtype=torch.float64))
    rows = torch.randn((196, 40), generator=torch.Generator().manual_seed(h * w), dtype=torch.float64)
    ref = F.interpolate(rows.t().reshape(1, 40, 14, 14), size=(h, w), mode="bicubic", antialias=True,
                        align_corners=False).reshape(40, h * w).t()
    assert float((M @ rows - ref).abs().max()) <= 1e-14 * float(ref.abs().max())


def test_patch_matrix_matches_normalize_and_conv2d_in_float64():
    from torchvision import transforms
    from oracle.vit_torch import MEAN, STD, patch_matrix
    img = images(2, 64, 48, 3).double()
    g = torch.Generator().manual_seed(4)
    w, b = torch.randn((40, 3, 16, 16), generator=g, dtype=torch.float64), torch.randn(40, generator=g,
                                                                                       dtype=torch.float64)
    ref = F.conv2d(transforms.Normalize(MEAN, STD)(img), w, b, stride=16)
    mine = (patch_matrix(img) @ w.view(40, -1).t() + b).transpose(1, 2).reshape(ref.shape)
    assert float((mine - ref).abs().max()) <= 1e-13 * float(ref.abs().max())


def test_restatement_matches_timm_when_timm_is_installed():
    timm = pytest.importorskip("timm")
    from oracle.vit_torch import normalize, vit_forward
    for C in sorted(WIDTHS):
        model = timm.create_model(NAMES[C], pretrained=False, dynamic_img_size=True).double().eval()
        p = {k: v.double() for k, v in vit_params(C, 12, 5).items()}
        model.load_state_dict(p, strict=True)
        img = images(1, 256, 192, 6).double()
        with torch.no_grad():
            ref = model.forward_features(normalize(img))[:, 1:]
            mine = vit_forward(img, p, WIDTHS[C])
        assert float((mine - ref).abs().max()) <= 1e-12 * float(ref.abs().max())


# ---- CPU: the module's surface -----------------------------------------------------------------------------------
@pytest.mark.parametrize("C", sorted(WIDTHS))
def test_state_dict_has_timms_keys_and_a_lara_checkpoint_loads_strictly(C):
    from lara_b200.image_encoder import DinoEncoder
    enc = DinoEncoder(NAMES[C], is_train=False)
    sd = enc.model.state_dict()
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == timm_keys(C)
    assert len(sd) == 150 and enc.model.num_features == C
    assert not any(p.requires_grad for p in enc.parameters()) and not enc.model.training
    enc.freeze(True)
    assert all(p.requires_grad for p in enc.parameters()) and enc.model.training
    p = vit_params(C, 12, 9)
    ckpt = {"net.img_encoder.model." + k: v for k, v in p.items()}
    ckpt["net.vol_decoder.norm.weight"] = torch.ones(3)
    loaded = DinoEncoder.from_lara_state_dict(ckpt, NAMES[C], is_train=True)
    assert all(torch.equal(loaded.model.state_dict()[k], v) for k, v in p.items())
    del ckpt["net.img_encoder.model.norm.bias"]
    with pytest.raises(RuntimeError, match="Missing key"):
        DinoEncoder.from_lara_state_dict(ckpt, NAMES[C])


def test_encoder_rejects_bad_names_sizes_dtypes_and_devices_before_any_launch():
    from lara_b200.image_encoder import DinoEncoder, patchify
    for name in ("vit_large_patch16_224.dino", "vit_base_patch16_224", "", None):
        with pytest.raises(ValueError, match="model_name"):
            DinoEncoder(name)
    enc = DinoEncoder(NAMES[384])
    for bad, msg in ((torch.zeros(1, 3, 40, 32), "multiples of 16"), (torch.zeros(1, 3, 0, 32), "multiples of 16"),
                     (torch.zeros(1, 4, 32, 32), "\\[N, 3, H, W\\]"), (torch.zeros(3, 32, 32), "\\[N, 3, H, W\\]"),
                     (torch.zeros(0, 3, 32, 32), "N >= 1"), ("image", "\\[N, 3, H, W\\]"),
                     (torch.zeros(1, 3, 32, 32, dtype=torch.float64), "Float"),
                     (torch.zeros(1, 3, 32, 32, dtype=torch.uint8), "Float"),
                     (torch.zeros(1, 3, 32, 32), "CUDA tensor")):
        with pytest.raises(RuntimeError, match=msg):
            enc(bad)
        with pytest.raises(RuntimeError, match=msg):
            patchify(bad)
    with pytest.raises(RuntimeError, match="constants"):
        enc(torch.zeros(1, 3, 32, 32, requires_grad=True))
    enc.model.double()
    with pytest.raises(RuntimeError, match="float32"):
        enc(torch.zeros(1, 3, 32, 32))


P = ctypes.c_void_p(256)                 # never dereferenced: the checks come before any CUDA call


def test_c_entries_reject_bad_arguments_before_any_launch(lib):
    size = ctypes.c_size_t()
    for N, H, W in ((0, 32, 32), (1, 40, 32), (1, 32, 8), (1, 0, 32), (-1, 32, 32)):
        assert lib.srf_vit_patchify(None, N, H, W, 0, 0, 0, 0, P, P) != 0
        assert b"srf_vit_patchify: bad sizes" in lib.srf_last_error()
    assert lib.srf_vit_patchify(None, 1, 32, 32, 0, 0, 0, 0, None, P) != 0
    assert b"null pointer" in lib.srf_last_error()
    for N, L, C, eps in ((0, 4, 768, 1e-6), (1, 0, 768, 1e-6), (1, 4, 512, 1e-6), (1, 4, 544, 1e-6), (1, 4, 768, 0.0),
                         (1, 4, 384, float("nan")), (2 ** 20, 2 ** 12, 768, 1e-6)):
        assert lib.srf_vit_tokens_forward(None, N, L, C, eps, *[P] * 9) != 0
        assert b"srf_vit_tokens_forward: bad" in lib.srf_last_error()
        assert lib.srf_vit_tokens_backward(None, N, L, C, eps, *[P] * 11) != 0
        assert b"srf_vit_tokens_backward: bad" in lib.srf_last_error()
        assert lib.srf_vit_final_norm_forward(None, N, L, C, eps, *[P] * 6) != 0
        assert b"srf_vit_final_norm_forward: bad" in lib.srf_last_error()
        assert lib.srf_vit_final_norm_backward(None, N, L, C, eps, *[P] * 7) != 0
        assert b"srf_vit_final_norm_backward: bad" in lib.srf_last_error()
    for rows, C, eps in ((-1, 768, 1e-6), (8, 256, 1e-6), (8, 544, 1e-6), (8, 768, 0.0)):
        assert lib.srf_vit_layernorm_forward(None, rows, C, eps, *[P] * 6) != 0
        assert b"srf_vit_layernorm_forward: bad" in lib.srf_last_error()
        assert lib.srf_vit_layernorm_backward(None, rows, C, eps, *[P] * 8) != 0
        assert b"srf_vit_layernorm_backward: bad" in lib.srf_last_error()
    assert lib.srf_vit_layernorm_workspace_bytes(8, 256, ctypes.byref(size)) != 0
    assert lib.srf_vit_tokens_workspace_bytes(12, 1024, 768, None) != 0
    assert lib.srf_vit_tokens_workspace_bytes(12, 1024, 768, ctypes.byref(size)) == 0
    assert size.value >= 1024 * 768 * 8 + 2 * 768 * 4 * (12 * 1025 // 64)
    assert lib.srf_vit_final_norm_workspace_bytes(12, 1024, 768, ctypes.byref(size)) == 0
    assert size.value >= 12 * 1025 * 768 * 4
    for k in range(9):
        ptrs = [P] * 9
        ptrs[k] = None
        assert lib.srf_vit_tokens_forward(None, 2, 4, 768, 1e-6, *ptrs) != 0
        assert b"null pointer" in lib.srf_last_error()
    assert lib.srf_vit_tokens_backward(None, 2, 4, 768, 1e-6, P, P, P, None, ctypes.c_void_p(264), *[P] * 6) != 0
    assert b"workspace must be 256-byte aligned" in lib.srf_last_error()
    assert lib.srf_vit_final_norm_backward(None, 2, 4, 768, 1e-6, P, P, P, P, P, None, P) != 0
    assert b"null gradient pointer" in lib.srf_last_error()
    assert lib.srf_vit_final_norm_forward(None, 2, 4, 768, 1e-6, P, None, P, P, None, P) != 0
    assert b"null pointer" in lib.srf_last_error()
    assert lib.srf_vit_layernorm_forward(None, 8, 768, 1e-6, P, P, P, P, None, P) != 0
    assert b"null y with a residual b" in lib.srf_last_error()


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


# N, H, W, C
KERNEL_CASES = {"lara": (12, 512, 512, 768), "one_image": (1, 512, 512, 768), "one_patch": (3, 16, 16, 768),
                "512x384": (2, 512, 384, 768), "c384": (4, 512, 512, 384)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(KERNEL_CASES))
def test_patchify_matches_float64_for_lara_view_and_contiguous_images(cuda_device, name):
    from lara_b200.image_encoder import patchify
    from oracle.vit_torch import patch_matrix
    N, H, W, _ = KERNEL_CASES[name]
    rgb = torch.rand((1, N, H, W, 3), generator=torch.Generator().manual_seed(N + H)).to(cuda_device)
    inps = torch.einsum("bhwc->bchw", rgb.reshape(N, H, W, 3))     # LaRa's _inps: a permuted view of tar_rgb
    assert not inps.is_contiguous()
    ref = patch_matrix(inps.double())
    view, contig = patchify(inps), patchify(inps.contiguous())
    assert torch.equal(view, contig)
    assert _err(view, ref) <= TOL, _err(view, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(KERNEL_CASES))
def test_tokens_and_final_norm_kernels_match_float64(cuda_device, name):
    from lara_b200.image_encoder import _FinalNorm, _Tokens
    N, H, W, C = KERNEL_CASES[name]
    h, w, dev = H // 16, W // 16, cuda_device
    L = h * w
    g = torch.Generator().manual_seed(N * C + L)
    t = {"patch_out": torch.randn((N, L, C), generator=g) * 2, "bias": 0.3 * torch.randn(C, generator=g),
         "cls": torch.randn(C, generator=g), "pos0": 0.5 * torch.randn(C, generator=g),
         "pos_r": 0.5 * torch.randn((L, C), generator=g), "gamma": 1 + 0.2 * torch.randn(C, generator=g),
         "beta": 0.1 * torch.randn(C, generator=g)}
    gx, gn = torch.randn((N, L + 1, C), generator=g).to(dev), torch.randn((N, L + 1, C), generator=g).to(dev)
    mine = {k: v.to(dev).requires_grad_(True) for k, v in t.items()}
    x, n1 = _Tokens.apply(*mine.values(), 1e-6)
    torch.autograd.backward([x, n1], [gx, gn])
    ref = {k: v.to(dev).double().requires_grad_(True) for k, v in t.items()}
    rx = torch.cat([(ref["cls"] + ref["pos0"]).expand(N, 1, C), (ref["patch_out"] + ref["bias"]) + ref["pos_r"]], 1)
    rn = F.layer_norm(rx, (C,), ref["gamma"], ref["beta"], 1e-6)
    torch.autograd.backward([rx, rn], [gx.double(), gn.double()])
    errs = {"x": _err(x.detach(), rx.detach()), "n1": _err(n1.detach(), rn.detach())}
    errs.update({"d_" + k: _err(mine[k].grad, ref[k].grad) for k in t})
    # the final norm: a, b [N, 1 + L, C] -> maps [N, C, h, w]
    a, b = (torch.randn((N, L + 1, C), generator=g).to(dev) for _ in range(2))
    gm = torch.randn((N, C, h, w), generator=g).to(dev)
    ai, bi = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    gam, bet = (mine["gamma"].detach().clone().requires_grad_(True), mine["beta"].detach().clone().requires_grad_(True))
    maps = _FinalNorm.apply(ai, bi, gam, bet, 1e-6, h, w, True)
    assert maps.shape == (N, C, h, w) and maps.is_contiguous()
    maps.backward(gm)
    ad, bd = a.double().requires_grad_(True), b.double().requires_grad_(True)
    gd, bed = gam.detach().double().requires_grad_(True), bet.detach().double().requires_grad_(True)
    rm = F.layer_norm(ad + bd, (C,), gd, bed, 1e-6)[:, 1:].transpose(1, 2).reshape(N, C, h, w)
    rm.backward(gm.double())
    errs.update({"maps": _err(maps.detach(), rm.detach()), "final_da": _err(ai.grad, ad.grad),
                 "final_dgamma": _err(gam.grad, gd.grad), "final_dbeta": _err(bet.grad, bed.grad)})
    assert torch.equal(ai.grad, bi.grad) and not ai.grad[:, 0].any()
    print(name, {k: f"{e:.2e}" for k, e in errs.items()})
    assert all(e <= TOL for e in errs.values()), errs


def _encoder_arms(dev, C, N, H, W, seed, arms, bf16=False):
    """{arm: {"out": [N, L, C], name: grad}} for the arms "fused", "fp32" (the restatement) and "f64"."""
    from lara_b200.image_encoder import DinoEncoder
    from oracle.vit_torch import vit_forward
    p = {k: v.to(dev) for k, v in vit_params(C, 12, seed).items()}
    img = images(N, H, W, seed + 1).to(dev)
    up = torch.randn((N, (H // 16) * (W // 16), C), generator=torch.Generator().manual_seed(seed + 2)).to(dev)
    res = {}
    for arm in arms:
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=bf16 and arm != "f64"):
            if arm == "fused":
                enc = DinoEncoder(NAMES[C], is_train=True).to(dev)
                enc.model.load_state_dict(p, strict=True)
                out = enc(img)
                named = dict(enc.model.named_parameters())
            else:
                cast = (lambda t: t.double()) if arm == "f64" else (lambda t: t)
                named = {k: cast(v).clone().requires_grad_(True) for k, v in p.items()}
                out = vit_forward(cast(img), named, WIDTHS[C])
        out.backward(up.to(out.dtype))
        res[arm] = {"out": out.detach(), **{k: t.grad for k, t in named.items()}}
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("C", sorted(WIDTHS))
def test_encoder_matches_float64_beside_the_fp32_restatement(cuda_device, no_tf32, C):
    res = _encoder_arms(cuda_device, C, 2, 512, 384, 21, ("f64", "fp32", "fused"))
    assert len(res["fused"]) == 151
    fp32 = {k: _err(res["fp32"][k], res["f64"][k]) for k in res["f64"]}
    mine = {k: _err(res["fused"][k], res["f64"][k]) for k in res["f64"]}
    print(f"C={C} worst error: fused {max(mine.values()):.2e}, fp32 restatement {max(fp32.values()):.2e}")
    # 2x the fp32 restatement's error per tensor, above fp32's rounding unit (2^-24 ~ 6e-8)
    bad = {k: (f"{mine[k]:.2e}", f"{fp32[k]:.2e}") for k in mine if not mine[k] <= max(2 * fp32[k], 6e-8)}
    assert bad == {}, bad
    res16 = _encoder_arms(cuda_device, C, 2, 512, 384, 21, ("fp32", "fused"), bf16=True)
    e16 = {arm: max(_err(res16[arm][k], res["f64"][k]) for k in res["f64"]) for arm in res16}
    e16_out = {arm: _err(res16[arm]["out"], res["f64"]["out"]) for arm in res16}
    print(f"C={C} bf16 autocast, worst error from float64 over the output and gradients: {e16}; output: {e16_out}")
    assert e16_out["fused"] <= max(2 * e16_out["fp32"], 1e-2)


def _fwd_bwd(enc, img, up, bf16):
    enc.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=bf16):
        out = enc(img)
    out.float().backward(up)
    return [out.detach()] + [p.grad.clone() for p in enc.parameters()]


@pytest.mark.gpu
@pytest.mark.parametrize("bf16", [False, True])
def test_encoder_is_bit_reproducible_under_the_deterministic_switch_and_no_grad_gives_the_same_bits(cuda_device, bf16):
    from lara_b200.image_encoder import DinoEncoder
    dev = cuda_device
    enc = DinoEncoder(NAMES[768], is_train=True).to(dev)
    enc.model.load_state_dict({k: v.to(dev) for k, v in vit_params(768, 12, 31).items()}, strict=True)
    img = images(3, 256, 256, 32).to(dev)
    up = torch.randn((3, 256, 768), generator=torch.Generator().manual_seed(33)).to(dev)
    was = torch.are_deterministic_algorithms_enabled()
    try:
        for det in (True, False):
            torch.use_deterministic_algorithms(det)
            runs = [_fwd_bwd(enc, img, up, bf16) for _ in range(2)] if det else [_fwd_bwd(enc, img, up, bf16)]
            if det:
                assert all(torch.equal(a, b) for a, b in zip(runs[0], runs[1]))
            for mode in (torch.no_grad, torch.inference_mode):
                with mode(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=bf16):
                    assert torch.equal(enc(img), runs[0][0]), (det, mode)
    finally:
        torch.use_deterministic_algorithms(was)


@pytest.mark.gpu
def test_chain_to_feat_volume_through_laras_einsum_and_reshape(cuda_device, no_tf32):
    from lara_b200.feat_volume import FeatVolume
    from lara_b200.image_encoder import DinoEncoder
    from oracle.vit_torch import img_feats as lara_img_feats, vit_forward
    from test_feat_volume import make_case
    dev, B, V, H, W, R, E = cuda_device, 1, 2, 256, 192, 16, 32
    p = {k: v.to(dev) for k, v in vit_params(768, 12, 41).items()}
    enc = DinoEncoder(NAMES[768], is_train=True).to(dev)
    enc.model.load_state_dict(p, strict=True)
    _, rays, w2c, ixt, params, ve = make_case(B, V, 768, H // 16, W // 16, H, W, R, E, 42)
    fv = FeatVolume(768, E, R).to(dev)
    with torch.no_grad():
        for t, v in zip((fv.dir_norm.norm.weight, fv.dir_norm.norm.bias, fv.dir_norm.mlp[1].weight,
                         fv.dir_norm.mlp[1].bias), params):
            t.copy_(v)
    rays, w2c, ixt = rays.to(dev), w2c.to(dev), ixt.to(dev)
    img = images(B * V, H, W, 43).to(dev)
    tokens = enc(img)
    feats = lara_img_feats(tokens, H, W)
    assert feats.is_contiguous() and feats.data_ptr() == tokens.data_ptr() and feats.shape == (B * V, 768, 16, 12)
    out = fv(feats, rays, w2c, ixt, (H, W))
    assert torch.equal(out, fv(feats.detach().clone(), rays, w2c, ixt, (H, W)))
    with torch.no_grad():
        ref = fv(lara_img_feats(vit_forward(img.double(), {k: v.double() for k, v in p.items()}, 12).float(), H, W)
                 .contiguous(), rays, w2c, ixt, (H, W))
    e = _err(out.detach(), ref)
    print(f"FeatVolume on the fused encoder's img_feats vs on the float64 restatement's: {e:.2e}")
    assert e <= 1e-4
    out.square().mean().backward()
    assert all(t.grad is not None and bool(torch.isfinite(t.grad).all()) for t in enc.parameters())
