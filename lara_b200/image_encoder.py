"""LaRa's image encoder (``DinoWrapper``, lightning/network.py:14-55, 442-445): timm's DINO ViT, ``vit_base_patch16_224
.dino`` (C = 768, 12 heads) or ``vit_small_patch16_224.dino`` (C = 384, 6 heads), under timm's parameter names, with
the patch and position embedding and the residual LayerNorms on the kernels of csrc/image_encoder.cu
(include/surfel_image_encoder.h).

The op sequence is timm's (written out in oracle/vit_torch.py and DESIGN §3.25).  Per image [3, H, W] in [0, 1]:

* ``srf_vit_patchify`` reads the image at any strides (LaRa's ``_inps`` is a permuted view of ``tar_rgb``), applies
  Normalize and writes the patch matrix; the patch conv is one GEMM on it (cuBLAS);
* ``srf_vit_tokens_*`` adds the conv bias and the position rows, puts the cls token first and runs block 0's
  ``norm1`` in the same pass.  ``pos_embed``'s patch rows are resampled to ``(H/16, W/16)`` by a ``[h w, 196]`` map
  built once per size in float64 from ``F.interpolate(mode='bicubic', antialias=True)`` of the 196 basis images (the
  op is linear, so the map is exact); its forward and backward are small GEMMs;
* each block hands ``(y, fc2_out)`` to the next un-added; the add fuses into the next ``norm1``, and ``norm2`` takes
  ``x + proj_out`` (``srf_vit_layernorm_*``);
* ``srf_vit_final_norm_*`` adds, normalises, drops the cls row and stores ``[N, C, h, w]`` contiguous, the layout
  ``FeatVolume`` reads.  ``forward`` returns it as LaRa's ``[N, h w, C]`` view, so LaRa's ``einsum('blc->bcl')`` and
  reshape give ``img_feats`` without a copy.

qkv, the attention core (``F.scaled_dot_product_attention``), proj and the MLP stay torch and follow autocast.  The
CUDA ops compute in fp32 (``custom_fwd(cast_inputs=torch.float32)``) and their backward uses no float atomics.  Under
``torch.use_deterministic_algorithms(True)`` torch's SDPA selection leaves out cuDNN attention, and the memory-efficient
(fp32) and flash (bf16) backends run their deterministic backward, so repeated forward + backward calls give
identical bits.

Differences from timm, by design: H and W must be multiples of 16 (timm's strided conv floors the size silently);
the images are constants (no gradient flows to them); only the two models above are built.
"""
from __future__ import annotations

import functools

import torch
import torch.nn.functional as F
from torch import nn

from . import _lib
from .vol_transformer import _AddLayerNorm

MODELS = {"vit_base_patch16_224.dino": (768, 12), "vit_small_patch16_224.dino": (384, 6)}
DEPTH = 12
PATCH = 16
GRID = 14                  # pos_embed's patch rows: 14 x 14 (224 / 16)
EPS = 1e-6
PATCH_K = 3 * PATCH * PATCH


@functools.lru_cache(maxsize=16)
def _resample_map64(h: int, w: int) -> torch.Tensor:
    basis = torch.eye(GRID * GRID, dtype=torch.float64).view(GRID * GRID, 1, GRID, GRID)
    out = F.interpolate(basis, size=(h, w), mode="bicubic", antialias=True, align_corners=False)
    return out.view(GRID * GRID, h * w).t().contiguous()


def resample_map(h: int, w: int) -> torch.Tensor:
    """The float64 ``[h w, 196]`` map M with ``M @ rows`` = ``F.interpolate(rows as [C, 14, 14], (h, w),
    mode='bicubic', antialias=True, align_corners=False)`` as ``[h w, C]``; the identity at 14 x 14."""
    return _resample_map64(int(h), int(w))


@functools.lru_cache(maxsize=16)
def _resample_map32(h: int, w: int, device: torch.device) -> torch.Tensor:
    return resample_map(h, w).to(device=device, dtype=torch.float32)


def patchify(image, fn="patchify"):
    """Normalize and cut [N, 3, H, W] fp32 CUDA images (any strides, H and W multiples of 16) into the patch matrix
    [N, h w, 3 16 16], columns in the patch conv weight's (c, ky, kx) order."""
    if not isinstance(image, torch.Tensor) or image.ndim != 4 or image.shape[1] != 3:
        raise RuntimeError(f"{fn}: image must be [N, 3, H, W], got "
                           f"{tuple(image.shape) if isinstance(image, torch.Tensor) else type(image)}")
    N, _, H, W = (int(s) for s in image.shape)
    if N < 1 or H < PATCH or W < PATCH or H % PATCH or W % PATCH:
        raise RuntimeError(f"{fn}: need N >= 1 and H, W positive multiples of {PATCH}, got {N} x {H} x {W}")
    if image.dtype != torch.float32:
        raise RuntimeError(f"{fn}: expected scalar type Float but found {image.dtype} for image")
    if not image.is_cuda:
        raise RuntimeError(f"{fn}: image must be a CUDA tensor, got {image.device}")
    out = torch.empty((N, (H // PATCH) * (W // PATCH), PATCH_K), device=image.device)
    _lib.launch("srf_vit_patchify", image.device, N, H, W, *image.stride(), image.data_ptr(), out.data_ptr())
    return out


class _Tokens(torch.autograd.Function):
    """(patch_out [N, L, C], bias, cls [C], pos0 [C], pos_r [L, C], gamma, beta, eps) -> (x, n1) [N, 1 + L, C]."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, patch_out, bias, cls, pos0, pos_r, gamma, beta, eps):
        patch_out, pos_r = patch_out.contiguous(), pos_r.contiguous()
        N, L, C = (int(s) for s in patch_out.shape)
        x = torch.empty((N, L + 1, C), device=patch_out.device)
        n1 = torch.empty_like(x)
        _lib.launch("srf_vit_tokens_forward", x.device, N, L, C, eps, patch_out.data_ptr(), bias.data_ptr(),
                    cls.data_ptr(), pos0.data_ptr(), pos_r.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                    x.data_ptr(), n1.data_ptr())
        ctx.save_for_backward(x, gamma)
        ctx.eps = eps
        return x, n1

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, gx, gn):
        x, gamma = ctx.saved_tensors
        N, T, C = (int(s) for s in x.shape)
        L = T - 1
        gn = gn.contiguous() if gn is not None else torch.zeros_like(x)
        gx = gx.contiguous() if gx is not None else None
        gt = torch.empty_like(x)
        d_bias, d_cls, d_gamma, d_beta = (torch.empty_like(gamma) for _ in range(4))
        d_pos_r = torch.empty((L, C), device=x.device)
        with _lib._DeviceGuard(x.device):
            nbytes = _lib.vit_tokens_workspace_bytes(_lib.load(), N, L, C)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
        _lib.launch("srf_vit_tokens_backward", x.device, N, L, C, ctx.eps, x.data_ptr(), gamma.data_ptr(),
                    gn.data_ptr(), gx.data_ptr() if gx is not None else None, ws.data_ptr(), gt.data_ptr(),
                    d_bias.data_ptr(), d_cls.data_ptr(), d_pos_r.data_ptr(), d_gamma.data_ptr(), d_beta.data_ptr())
        return gt[:, 1:], d_bias, d_cls, d_cls, d_pos_r, d_gamma, d_beta, None


class _FinalNorm(torch.autograd.Function):
    """(a, b [N, 1 + L, C], gamma, beta, eps, h, w, keep_y) -> maps [N, C, h, w] = LN(a + b) without the cls row."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, a, b, gamma, beta, eps, h, w, keep_y):
        a, b = a.contiguous(), b.contiguous()
        N, T, C = (int(s) for s in a.shape)
        maps = torch.empty((N, C, h, w), device=a.device)
        y = torch.empty_like(a) if keep_y else None
        _lib.launch("srf_vit_final_norm_forward", a.device, N, T - 1, C, eps, a.data_ptr(), b.data_ptr(),
                    gamma.data_ptr(), beta.data_ptr(), y.data_ptr() if y is not None else None, maps.data_ptr())
        if keep_y:
            ctx.save_for_backward(y, gamma)
        ctx.eps = eps
        return maps

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, gm):
        y, gamma = ctx.saved_tensors
        N, T, C = (int(s) for s in y.shape)
        gm = gm.contiguous()
        ga = torch.empty_like(y)
        d_gamma, d_beta = torch.empty_like(gamma), torch.empty_like(gamma)
        with _lib._DeviceGuard(y.device):
            nbytes = _lib.vit_final_norm_workspace_bytes(_lib.load(), N, T - 1, C)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=y.device)
        _lib.launch("srf_vit_final_norm_backward", y.device, N, T - 1, C, ctx.eps, y.data_ptr(), gamma.data_ptr(),
                    gm.data_ptr(), ws.data_ptr(), ga.data_ptr(), d_gamma.data_ptr(), d_beta.data_ptr())
        return ga, ga, d_gamma, d_beta, None, None, None, None


class PatchEmbed(nn.Module):
    """timm's ``patch_embed``: only its ``proj`` conv's parameters."""

    def __init__(self, C: int):
        super().__init__()
        self.proj = nn.Conv2d(3, C, kernel_size=PATCH, stride=PATCH)


class Attention(nn.Module):
    def __init__(self, C: int):
        super().__init__()
        self.qkv = nn.Linear(C, 3 * C)
        self.proj = nn.Linear(C, C)


class Mlp(nn.Module):
    def __init__(self, C: int):
        super().__init__()
        self.fc1 = nn.Linear(C, 4 * C)
        self.fc2 = nn.Linear(4 * C, C)


class Block(nn.Module):
    def __init__(self, C: int):
        super().__init__()
        self.norm1 = nn.LayerNorm(C, eps=EPS)
        self.attn = Attention(C)
        self.norm2 = nn.LayerNorm(C, eps=EPS)
        self.mlp = Mlp(C)


class VisionTransformer(nn.Module):
    """The parameters of timm's ``VisionTransformer`` for the DINO models, under timm's names and shapes:
    ``cls_token``, ``pos_embed``, ``patch_embed.proj``, ``blocks.{i}.{norm1, attn.qkv, attn.proj, norm2, mlp.fc1,
    mlp.fc2}`` and ``norm`` (150 tensors).  The initialisation is not timm's random draw: weights come from LaRa's
    checkpoint or from a timm model's ``state_dict``."""

    def __init__(self, C: int, num_heads: int, depth: int = DEPTH):
        super().__init__()
        self.num_features = self.embed_dim = C
        self.num_heads = num_heads
        self.cls_token = nn.Parameter(torch.randn(1, 1, C) * 1e-6)
        self.pos_embed = nn.Parameter(torch.randn(1, 1 + GRID * GRID, C) * 0.02)
        self.patch_embed = PatchEmbed(C)
        self.blocks = nn.ModuleList([Block(C) for _ in range(depth)])
        self.norm = nn.LayerNorm(C, eps=EPS)


def _attention(blk: Block, n1, heads: int):
    N, T, C = n1.shape
    qkv = blk.attn.qkv(n1).reshape(N, T, 3, heads, C // heads).permute(2, 0, 3, 1, 4)
    q, k, v = qkv.unbind(0)
    o = F.scaled_dot_product_attention(q, k, v)
    return blk.attn.proj(o.transpose(1, 2).reshape(N, T, C))


class DinoEncoder(nn.Module):
    """``DinoWrapper`` with the same surface: ``DinoEncoder(model_name, is_train)``, ``.model`` (timm's names and
    ``num_features``), ``freeze(is_train)`` and ``forward(image [N, 3, H, W] in [0, 1]) -> [N, h w, C]``."""

    def __init__(self, model_name: str, is_train: bool = False):
        super().__init__()
        if model_name not in MODELS:
            raise ValueError(f"DinoEncoder: model_name must be one of {sorted(MODELS)}, got {model_name!r}")
        self.model_name = model_name
        C, heads = MODELS[model_name]
        self.model = VisionTransformer(C, heads)
        self.freeze(is_train)

    def freeze(self, is_train: bool = False):
        self.model.train(is_train)
        for p in self.model.parameters():
            p.requires_grad = is_train

    @classmethod
    def from_lara_state_dict(cls, sd, model_name: str = "vit_base_patch16_224.dino", is_train: bool = False):
        """The encoder of a LaRa checkpoint's state dict: its ``net.img_encoder.model.*`` entries, loaded strictly."""
        prefix = "net.img_encoder.model."
        enc = cls(model_name, is_train)
        enc.model.load_state_dict({k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}, strict=True)
        return enc

    def forward(self, image):
        """image [N, 3, H, W] in [0, 1], H and W multiples of 16 -> [N, h w, C], a transposed view of the contiguous
        ``[N, C, h, w]`` maps of :meth:`forward_maps`."""
        return self.forward_maps(image).flatten(2).transpose(1, 2)

    def forward_maps(self, image):
        """image [N, 3, H, W] -> [N, C, h, w] contiguous: LaRa's ``img_feats``."""
        fn = "DinoEncoder.forward"
        m = self.model
        C, heads, dev = m.num_features, m.num_heads, m.cls_token.device
        for name, t in m.named_parameters():
            if t.dtype != torch.float32 or t.device != dev:
                raise RuntimeError(f"{fn}: parameter {name} must be float32 on {dev}, got {t.dtype} on {t.device}")
        if isinstance(image, torch.Tensor) and image.device != dev:
            raise RuntimeError(f"{fn}: image must be a CUDA tensor on {dev}, got {image.device}")
        if isinstance(image, torch.Tensor) and image.requires_grad and torch.is_grad_enabled():
            raise RuntimeError(f"{fn}: the images are constants; no gradient flows to them")
        P = patchify(image, fn)
        N, H, W = int(image.shape[0]), int(image.shape[2]), int(image.shape[3])
        h, w = H // PATCH, W // PATCH
        grad = torch.is_grad_enabled() and any(p.requires_grad for p in m.parameters())
        patch_out = F.linear(P, m.patch_embed.proj.weight.view(C, PATCH_K))
        pos = m.pos_embed[0]
        if (h, w) == (GRID, GRID):
            pos_r = pos[1:]
        else:
            with torch.autocast("cuda", enabled=False):
                pos_r = _resample_map32(h, w, dev) @ pos[1:]
        b0 = m.blocks[0]
        x, n1 = _Tokens.apply(patch_out, m.patch_embed.proj.bias, m.cls_token.view(C), pos[0], pos_r,
                              b0.norm1.weight, b0.norm1.bias, EPS)
        for i, blk in enumerate(m.blocks):
            if i:
                x, n1 = _AddLayerNorm.apply(y, f, blk.norm1.weight, blk.norm1.bias, EPS, "srf_vit_layernorm")
            y, n2 = _AddLayerNorm.apply(x, _attention(blk, n1, heads), blk.norm2.weight, blk.norm2.bias, EPS,
                                        "srf_vit_layernorm")
            f = blk.mlp.fc2(F.gelu(blk.mlp.fc1(n2)))
        return _FinalNorm.apply(y, f, m.norm.weight, m.norm.bias, EPS, h, w, grad)


__all__ = ["DinoEncoder", "VisionTransformer", "MODELS", "patchify", "resample_map"]
