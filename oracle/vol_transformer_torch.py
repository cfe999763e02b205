"""Plain-torch restatements of LaRa's volume transformer (``GroupAttBlock.forward``, lightning/network.py:81-102, and
``VolTransformer.forward``, :138-164), the checkers of lara_b200/csrc/vol_transformer.cu.

* ``group_att_block_torch`` / ``vol_transformer_torch`` follow LaRa's layout and op sequence: the ``unfold`` /
  ``einsum`` groups, the op sequence ``nn.MultiheadAttention(C, H, kdim=vdim=Cc, bias=False, batch_first=True)``
  executes (``F.multi_head_attention_forward`` with separate projection weights and ``need_weights=False``: sequence-first
  projections and ``F.scaled_dot_product_attention``), the LayerNorms, the MLP and the convolutions.  On the CPU in fp32
  they reproduce LaRa's values and every gradient bit for bit (tests/test_vol_transformer.py).
* ``group_att_block_cl`` / ``vol_transformer_cl`` are the same computation on a channels-last volume [B,R,R,R,C], with
  the attention written out as ``softmax(q k^T / sqrt(D)) v`` per group.  In float64 they equal the LaRa-layout
  restatement to rounding and are the accuracy reference of the kernels.

``p`` is a parameter dict under LaRa's names relative to the block (``norm1.weight``, ``cross_attn.q_proj_weight``,
``mlp.0.weight``, ``cnn.weight``, ...) or the transformer (``pos_embed``, ``layers.0.norm1.weight``, ``norm.weight``,
``deconv.weight``, ...).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

BLOCK_EPS = 1e-5        # GroupAttBlock's norm_layer(inner_dim): LayerNorm's default eps (the eps argument is unused)


def _sub(p, prefix):
    return {k[len(prefix):]: v for k, v in p.items() if k.startswith(prefix)}


def cross_attn_torch(x, cond, p, H):
    """nn.MultiheadAttention(C, H, kdim=vdim=Cc, bias=False, batch_first=True)(x, cond, cond)[0]: x [N,L,C],
    cond [N,S,Cc] -> [N,L,C]."""
    N, L, C = x.shape
    hd = C // H
    query, key = x.transpose(1, 0), cond.transpose(1, 0)          # batch_first, key is value
    q = F.linear(query, p["cross_attn.q_proj_weight"])
    k = F.linear(key, p["cross_attn.k_proj_weight"])
    v = F.linear(key, p["cross_attn.v_proj_weight"])
    S = k.shape[0]
    q = q.view(L, N * H, hd).transpose(0, 1).view(N, H, L, hd)
    k = k.view(S, N * H, hd).transpose(0, 1).view(N, H, S, hd)
    v = v.view(S, N * H, hd).transpose(0, 1).view(N, H, S, hd)
    o = F.scaled_dot_product_attention(q, k, v)
    o = o.permute(2, 0, 1, 3).contiguous().view(N * L, C)
    o = F.linear(o, p["cross_attn.out_proj.weight"]).view(L, N, C)
    return o.transpose(1, 0)


def _ln(x, p, name, eps=BLOCK_EPS):
    return F.layer_norm(x, (x.shape[-1],), p[name + ".weight"], p[name + ".bias"], eps)


def _mlp(x, p):
    return F.linear(F.gelu(F.linear(x, p["mlp.0.weight"], p["mlp.0.bias"])), p["mlp.3.weight"], p["mlp.3.bias"])


def group_att_block_torch(x, cond, group_axis, block_size, p, H):
    """GroupAttBlock.forward: x [B,C,D,H,W], cond [B g^3, S, Cc] -> [B,C,D,H,W]."""
    B, C, D, Hh, W = x.shape
    patches = x.unfold(2, block_size, block_size).unfold(3, block_size, block_size).unfold(4, block_size, block_size)
    patches = patches.reshape(B, C, -1, block_size ** 3)
    patches = torch.einsum("bcgl->bglc", patches).reshape(B * group_axis ** 3, block_size ** 3, C)
    patches = patches + cross_attn_torch(_ln(patches, p, "norm1"), cond, p, H)
    patches = patches + _mlp(_ln(patches, p, "norm2"), p)
    patches = _ln(patches, p, "norm3")
    patches = patches.view(B, group_axis, group_axis, group_axis, block_size, block_size, block_size, C)
    patches = torch.einsum("bdhwzyxc->bcdzhywx", patches).reshape(x.shape)
    return patches + F.conv3d(patches, p["cnn.weight"], None, padding=1)


def cond_blocks_torch(image_feats, n_group):
    """VolTransformer.forward's condition blocks (:145-150): [B,V,Cc,D,D,D] -> [B g^3, V bs^3, Cc]."""
    B, V, C, D, _, _ = image_feats.shape
    bs = D // n_group
    blocks = image_feats.unfold(3, bs, bs).unfold(4, bs, bs).unfold(5, bs, bs)
    blocks = blocks.contiguous().view(B, V, C, n_group ** 3, bs ** 3)
    return torch.einsum("bvcgl->bgvlc", blocks).reshape(B * n_group ** 3, bs ** 3 * V, C)


def vol_transformer_torch(image_feats, p, n_groups, H, R, eps=1e-6):
    """VolTransformer.forward: image_feats [B,V,Cc,D,D,D] -> x_up [B,2R,2R,2R,out_dim] (contiguous)."""
    B = image_feats.shape[0]
    conds = [cond_blocks_torch(image_feats, g) for g in n_groups]
    x = p["pos_embed"].repeat(B, 1, 1, 1, 1)
    layers = sorted({int(k.split(".")[1]) for k in p if k.startswith("layers.")})
    for i in layers:
        gi = i % len(n_groups)
        x = group_att_block_torch(x, conds[gi], n_groups[gi], R // n_groups[gi], _sub(p, f"layers.{i}."), H)
    x = F.layer_norm(torch.einsum("bcdhw->bdhwc", x), (x.shape[1],), p["norm.weight"], p["norm.bias"], eps)
    x = torch.einsum("bdhwc->bcdhw", x)
    x_up = F.conv_transpose3d(x, p["deconv.weight"], p["deconv.bias"], stride=2)
    return torch.einsum("bcdhw->bdhwc", x_up).contiguous()


# ---- channels-last restatement ------------------------------------------------------------------------------------
def to_groups(x_cl, g):
    """[B,R,R,R,C] -> [B g^3, bs^3, C], group and in-group order of LaRa's unfold."""
    B, R, _, _, C = x_cl.shape
    bs = R // g
    return x_cl.reshape(B, g, bs, g, bs, g, bs, C).permute(0, 1, 3, 5, 2, 4, 6, 7).reshape(B * g ** 3, bs ** 3, C)


def from_groups(x_g, B, R, g):
    bs, C = R // g, x_g.shape[-1]
    return x_g.reshape(B, g, g, g, bs, bs, bs, C).permute(0, 1, 4, 2, 5, 3, 6, 7).reshape(B, R, R, R, C)


def group_attention_cl(q, k, v, g, H):
    """The attention core: q [B,R,R,R,C], k, v [B g^3, S, C] (projected) -> o [B,R,R,R,C]."""
    B, R, C = q.shape[0], q.shape[1], q.shape[-1]
    hd = C // H
    qg = to_groups(q, g)
    G, L, S = qg.shape[0], qg.shape[1], k.shape[1]
    qh = qg.view(G, L, H, hd).transpose(1, 2)
    kh = k.view(G, S, H, hd).transpose(1, 2)
    vh = v.view(G, S, H, hd).transpose(1, 2)
    s = qh @ kh.transpose(-1, -2) / hd ** 0.5
    o = torch.softmax(s, dim=-1) @ vh
    return from_groups(o.transpose(1, 2).reshape(G, L, C), B, R, g)


def group_att_block_cl(x_cl, cond, g, p, H):
    """GroupAttBlock on x_cl [B,R,R,R,C] with cond [B g^3, S, Cc] -> [B,R,R,R,C]."""
    q = F.linear(_ln(x_cl, p, "norm1"), p["cross_attn.q_proj_weight"])
    k = F.linear(cond, p["cross_attn.k_proj_weight"])
    v = F.linear(cond, p["cross_attn.v_proj_weight"])
    y = x_cl + F.linear(group_attention_cl(q, k, v, g, H), p["cross_attn.out_proj.weight"])
    n3 = _ln(y + _mlp(_ln(y, p, "norm2"), p), p, "norm3")
    return n3 + F.conv3d(n3.permute(0, 4, 1, 2, 3), p["cnn.weight"], None, padding=1).permute(0, 2, 3, 4, 1)


def vol_transformer_cl(conds, p, n_groups, H, B, eps=1e-6):
    """VolTransformer on the condition blocks (one per n_groups entry) -> x_up [B,2R,2R,2R,out_dim]."""
    x = p["pos_embed"].permute(0, 2, 3, 4, 1).expand(B, -1, -1, -1, -1)
    layers = sorted({int(k.split(".")[1]) for k in p if k.startswith("layers.")})
    for i in layers:
        gi = i % len(n_groups)
        x = group_att_block_cl(x, conds[gi], n_groups[gi], _sub(p, f"layers.{i}."), H)
    x = F.layer_norm(x, (x.shape[-1],), p["norm.weight"], p["norm.bias"], eps)
    x_up = F.conv_transpose3d(x.permute(0, 4, 1, 2, 3), p["deconv.weight"], p["deconv.bias"], stride=2)
    return x_up.permute(0, 2, 3, 4, 1)
