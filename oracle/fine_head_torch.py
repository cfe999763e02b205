"""Plain-torch restatement of LaRa's fine-pass decoder head (``Decoder.forward_fine``, lightning/network.py:280-284:
``norm`` -> ``cross_att`` -> ``mlp_fine``), the checker of lara_b200/csrc/fine_head.cu.

The op sequence is the one ``nn.MultiheadAttention(D, 8, kdim=8, vdim=8, bias=False, batch_first=True)`` executes
(``F.multi_head_attention_forward`` with separate projection weights and ``need_weights=False``): k and v are
projected from the sequence-first point features, and the attention is ``F.scaled_dot_product_attention``.  On the CPU
this reproduces LaRa's values and every gradient bit for bit (tests/test_fine_head.py); projecting k and v batch-first,
or an explicit ``softmax(q k^T / sqrt(d)) v``, does not.  In float64 it is the accuracy reference of the kernels.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

HEADS = 8


def fine_head_torch(volume_feat, point_feats, params):
    """volume_feat [n,D], point_feats [n,V,8] (batch-first, what forward_fine receives), params the ten tensors
    (norm weight, norm bias, Wq, Wk, Wv, Wo, W1, b1, W2, b2) -> sh [n,1,sh_dim]."""
    ln_w, ln_b, wq, wk, wv, wo, w1, b1, w2, b2 = params
    n, D = volume_feat.shape
    hd = D // HEADS
    x = F.layer_norm(volume_feat.unsqueeze(1), (D,), ln_w, ln_b, 1e-5)        # [n,1,D]
    query = x.transpose(0, 1)                                                  # [1,n,D] sequence-first
    kv = point_feats.transpose(0, 1)                                           # [V,n,8]
    q = F.linear(query, wq)
    k = F.linear(kv, wk)
    v = F.linear(kv, wv)
    V = k.shape[0]
    q = q.view(1, n * HEADS, hd).transpose(0, 1).view(n, HEADS, 1, hd)
    k = k.view(V, n * HEADS, hd).transpose(0, 1).view(n, HEADS, V, hd)
    v = v.view(V, n * HEADS, hd).transpose(0, 1).view(n, HEADS, V, hd)
    o = F.scaled_dot_product_attention(q, k, v)                                # [n,H,1,hd]
    o = o.permute(2, 0, 1, 3).contiguous().view(n, D)
    y = F.linear(o, wo).view(1, n, D).transpose(1, 0)                          # [n,1,D]
    return F.linear(F.relu(F.linear(y, w1, b1)), w2, b2)      # LaRa's .float() is a no-op in fp32


def fine_shs_torch(volume_feat_up, K, mask, point_feats, shs_coarse, params):
    """network.py:508-512 around the head: point_feats [V,8,n] -> _shs_fine [n,M,3]."""
    pf = torch.einsum("lcb->blc", point_feats)
    vpf = volume_feat_up.unsqueeze(1).expand(-1, K, -1)[mask.view(-1, K)]
    return fine_head_torch(vpf, pf, params).view(-1, *shs_coarse.shape[-2:]) + shs_coarse[mask]
