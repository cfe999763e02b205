"""timm's DINO ViT as LaRa's ``DinoWrapper`` runs it (lightning/network.py:14-55: ``vit_base_patch16_224.dino`` or
``vit_small_patch16_224.dino`` built with ``dynamic_img_size=True``, behind ``transforms.Normalize``), restated in torch
op by op.  Test-only: the kernels' reference, runnable in float64, and the fp32 arm of tools/bench_image_encoder.py.

The contract (DESIGN §3.25), on parameters under timm's names:

* Normalize: ``(x - mean) / std`` with ``mean = (0.485, 0.456, 0.406)``, ``std = (0.229, 0.224, 0.225)``;
* patch embed: ``Conv2d(3, C, 16, stride 16)`` with bias;
* tokens: ``cat(cls_token, patches) + pos_embed``, ``pos_embed``'s 196 patch rows resampled from 14 x 14 to
  ``(H/16, W/16)`` by ``F.interpolate(mode='bicubic', antialias=True, align_corners=False)`` in fp32 (float64 stays
  float64 here); the cls row is not resampled, and at 14 x 14 the rows are used unchanged;
* 12 blocks ``x = x + proj(SDPA(qkv(LN1(x))))``, ``x = x + fc2(GELU(fc1(LN2(x))))``: LayerNorm eps 1e-6, qkv with a
  bias splitting as ``[3, heads, 64]``, exact (erf) GELU, no LayerScale;
* the final ``norm`` (eps 1e-6), then ``outputs[:, 1:]``.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
EPS = 1e-6
PATCH = 16
GRID = 14                  # pos_embed's patch rows: 14 x 14 (224 / 16)


def normalize(image):
    """``transforms.Normalize(MEAN, STD)``: two elementwise operations in the image's dtype."""
    mean = torch.tensor(MEAN, dtype=image.dtype, device=image.device).view(1, 3, 1, 1)
    std = torch.tensor(STD, dtype=image.dtype, device=image.device).view(1, 3, 1, 1)
    return (image - mean) / std


def resample_pos_embed(pos_embed, h: int, w: int):
    """timm's ``resample_abs_pos_embed(pos_embed, (h, w), num_prefix_tokens=1)``: [1, 1 + 196, C] -> [1, 1 + h w, C]."""
    if (h, w) == (GRID, GRID):
        return pos_embed
    C, dt = pos_embed.shape[-1], pos_embed.dtype
    grid = pos_embed[:, 1:].reshape(1, GRID, GRID, C).permute(0, 3, 1, 2)
    grid = grid.to(torch.float64 if dt == torch.float64 else torch.float32)
    grid = F.interpolate(grid, size=(h, w), mode="bicubic", antialias=True, align_corners=False)
    grid = grid.permute(0, 2, 3, 1).reshape(1, h * w, C).to(dt)
    return torch.cat([pos_embed[:, :1], grid], dim=1)


def patch_matrix(image):
    """The normalised images as the patch matrix [N, h w, 3 16 16], row (n, py, px), column (c, ky, kx): the patch conv
    is ``patch_matrix(image) @ weight.view(C, -1).T + bias``."""
    N, _, H, W = image.shape
    x = normalize(image).reshape(N, 3, H // PATCH, PATCH, W // PATCH, PATCH)
    return x.permute(0, 2, 4, 1, 3, 5).reshape(N, (H // PATCH) * (W // PATCH), 3 * PATCH * PATCH)


def patch_tokens(image, p):
    """Normalize, the patch conv and the tokens with their position rows: [N, 3, H, W] -> [N, 1 + h w, C]."""
    x = F.conv2d(normalize(image), p["patch_embed.proj.weight"], p["patch_embed.proj.bias"], stride=PATCH)
    N, C, h, w = x.shape
    x = x.flatten(2).transpose(1, 2)
    x = torch.cat([p["cls_token"].expand(N, -1, -1).to(x.dtype), x], dim=1)
    return x + resample_pos_embed(p["pos_embed"], h, w)


def block(x, p, prefix: str, heads: int, eps: float = EPS):
    """One of timm's ``Block``s: pre-norm attention and MLP, each added to the residual stream."""
    N, T, C = x.shape
    n = F.layer_norm(x, (C,), p[prefix + "norm1.weight"], p[prefix + "norm1.bias"], eps)
    qkv = F.linear(n, p[prefix + "attn.qkv.weight"], p[prefix + "attn.qkv.bias"])
    q, k, v = qkv.reshape(N, T, 3, heads, C // heads).permute(2, 0, 3, 1, 4).unbind(0)
    o = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(N, T, C)
    x = x + F.linear(o, p[prefix + "attn.proj.weight"], p[prefix + "attn.proj.bias"])
    n = F.layer_norm(x, (C,), p[prefix + "norm2.weight"], p[prefix + "norm2.bias"], eps)
    m = F.gelu(F.linear(n, p[prefix + "mlp.fc1.weight"], p[prefix + "mlp.fc1.bias"]))
    return x + F.linear(m, p[prefix + "mlp.fc2.weight"], p[prefix + "mlp.fc2.bias"])


def depth(p) -> int:
    return sum(1 for k in p if k.startswith("blocks.") and k.endswith(".norm1.weight"))


def vit_forward(image, p, heads: int, eps: float = EPS):
    """``DinoWrapper.forward``: image [N, 3, H, W] in [0, 1] -> [N, h w, C] (the cls row dropped)."""
    x = patch_tokens(image, p)
    for i in range(depth(p)):
        x = block(x, p, f"blocks.{i}.", heads, eps)
    C = x.shape[-1]
    return F.layer_norm(x, (C,), p["norm.weight"], p["norm.bias"], eps)[:, 1:]


def img_feats(tokens, H: int, W: int):
    """LaRa's lines 443-445: ``einsum('blc->bcl')`` and the reshape to [N, C, H/16, W/16]."""
    f = torch.einsum("blc->bcl", tokens)
    return f.reshape(*f.shape[:2], H // PATCH, W // PATCH)
