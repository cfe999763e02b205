"""LaRa's volume transformer (``GroupAttBlock`` and ``VolTransformer``, lightning/network.py:57-164) on a channels-last
volume, with the group cross-attention core and the residual add + LayerNorms on the kernels of
csrc/vol_transformer.cu (include/surfel_vol_transformer.h).

The volume stays ``[B,R,R,R,C]`` from the first block to the ``deconv``.  Every op but two is then row-wise: the
LayerNorms, the projections, the residuals and the MLP.  The attention only needs each voxel's group, which the
kernel computes from its coordinates; the convolutions take the same memory as a ``channels_last_3d`` view.  So
LaRa's ``unfold`` / ``einsum`` copies and their gradients disappear.  The projections, the MLP and the
(de)convolutions stay plain torch (cuBLAS / cuDNN) and follow autocast as LaRa's do.  The CUDA ops compute in fp32
under autocast (``custom_fwd(cast_inputs=torch.float32)``).  Their backward uses no float atomics, so repeated calls
give identical bits whether or not ``torch.use_deterministic_algorithms`` is on (DESIGN §3.19).

The modules carry LaRa's parameter names and shapes, so ``VolTransformer.load_state_dict(net.vol_decoder
.state_dict())`` is strict.  Each block's ``norm3`` output and its convolution are handed to the next block
un-added: the add is fused into that block's ``norm1`` (or the final ``norm``).

Differences from LaRa, by design: no attention dropout or biases (LaRa has neither), ``cond_dim`` must differ from
``inner_dim`` (as in LaRa, where it selects ``nn.MultiheadAttention``'s separate projection weights), and
``GroupAttBlock.forward`` returns its ``[B,C,D,H,W]`` result in ``channels_last_3d`` memory format (and in fp32 under
bf16 autocast, where LaRa's closing ``einsum`` returns bf16).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch import nn

from . import _lib

BLOCK_EPS = 1e-5        # LaRa's norm_layer(inner_dim): LayerNorm's default eps


def _check_cuda_float(fn, named):
    autocast = torch.is_autocast_enabled("cuda")
    dev = named[0][1].device
    for name, t in named:
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{fn}: {name} must be a tensor")
        if not t.is_floating_point() or (not autocast and t.dtype != torch.float32):
            raise RuntimeError(f"{fn}: expected scalar type Float but found {t.dtype} for {name}")
        if not t.is_cuda or t.device != dev:
            raise RuntimeError(f"{fn}: {name} must be a CUDA tensor on {dev}, got {t.device}")


class _GroupAttn(torch.autograd.Function):
    """(q [B,R,R,R,C], k, v [B g^3, S, C], g, H) -> o [B,R,R,R,C]."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, q, k, v, g, H):
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        B, R, C, S = int(q.shape[0]), int(q.shape[1]), int(q.shape[-1]), int(k.shape[1])
        o = torch.empty_like(q)
        ctx.dims = (B, R, g, S, C, H)
        _lib.launch("srf_group_attn_forward", q.device, *ctx.dims, q.data_ptr(), k.data_ptr(), v.data_ptr(),
                    o.data_ptr())
        ctx.save_for_backward(q, k, v)
        return o

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, go):
        q, k, v = ctx.saved_tensors
        go = go.contiguous()
        gq, gk, gv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        _lib.launch("srf_group_attn_backward", q.device, *ctx.dims, q.data_ptr(), k.data_ptr(), v.data_ptr(),
                    go.data_ptr(), gq.data_ptr(), gk.data_ptr(), gv.data_ptr())
        return gq, gk, gv, None, None


class _AddLayerNorm(torch.autograd.Function):
    """(a, b or None, gamma, beta, eps, entry) -> (y = a + b, n = LN(y)), or n = LN(a) when b is None, on the C entries
    ``{entry}_forward`` / ``_workspace_bytes`` / ``_backward``: ``srf_add_layernorm`` (C <= 512) or
    ``srf_vit_layernorm`` (C in {384, 768})."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, a, b, gamma, beta, eps, entry="srf_add_layernorm"):
        a = a.contiguous()
        C = int(a.shape[-1])
        rows = a.numel() // C
        n = torch.empty_like(a)
        y = torch.empty_like(a) if b is not None else None
        if b is not None:
            b = b.contiguous()
        _lib.launch(entry + "_forward", a.device, rows, C, eps, a.data_ptr(),
                    b.data_ptr() if b is not None else None, gamma.data_ptr(), beta.data_ptr(),
                    y.data_ptr() if y is not None else None, n.data_ptr())
        ctx.save_for_backward(y if y is not None else a, gamma)
        ctx.eps, ctx.has_b, ctx.entry = eps, b is not None, entry
        return (y, n) if b is not None else n

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, *grads):
        y, gamma = ctx.saved_tensors
        gy, gn = grads if ctx.has_b else (None, grads[0])
        C = int(y.shape[-1])
        rows = y.numel() // C
        gn = gn.contiguous() if gn is not None else torch.zeros_like(y)
        gy = gy.contiguous() if gy is not None else None
        ga = torch.empty_like(y)
        g_gamma, g_beta = torch.empty_like(gamma), torch.empty_like(gamma)
        with _lib._DeviceGuard(y.device):
            nbytes = _lib.layernorm_workspace_bytes(_lib.load(), ctx.entry, rows, C)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=y.device)
        _lib.launch(ctx.entry + "_backward", y.device, rows, C, ctx.eps, y.data_ptr(), gamma.data_ptr(),
                    gn.data_ptr(), gy.data_ptr() if gy is not None else None, ws.data_ptr(), ga.data_ptr(),
                    g_gamma.data_ptr(), g_beta.data_ptr())
        return ga, (ga if ctx.has_b else None), g_gamma, g_beta, None, None


def add_layer_norm(a, b, norm: nn.LayerNorm, fn="add_layer_norm"):
    """``(a + b, norm(a + b))`` for ``b`` a tensor, ``norm(a)`` for ``b`` None, over the last dimension, on the
    kernels.  ``norm`` is an ``nn.LayerNorm`` over that dimension, with its weight and bias."""
    C = int(a.shape[-1]) if isinstance(a, torch.Tensor) else -1
    if C % 32 != 0 or not 32 <= C <= 512:
        raise RuntimeError(f"{fn}: the normalised dimension must be a multiple of 32 up to 512, got {C}")
    if tuple(norm.normalized_shape) != (C,) or norm.weight is None or norm.bias is None:
        raise RuntimeError(f"{fn}: norm must be an affine LayerNorm({C})")
    named = [("a", a)] + ([("b", b)] if b is not None else [])
    _check_cuda_float(fn, named)
    if b is not None and b.shape != a.shape:
        raise RuntimeError(f"{fn}: b must have a's shape {tuple(a.shape)}, got {tuple(b.shape)}")
    for name, t in (("norm.weight", norm.weight), ("norm.bias", norm.bias)):
        if t.dtype != torch.float32 or t.device != a.device:
            raise RuntimeError(f"{fn}: {name} must be float32 on {a.device}")
    return _AddLayerNorm.apply(a, b, norm.weight, norm.bias, float(norm.eps))


def group_attention(q, k, v, n_group: int, num_heads: int, fn="group_attention"):
    """The attention core of ``GroupAttBlock``: q [B,R,R,R,C] (projected, channels-last), k, v [B g^3, S, C]
    (projected) -> o [B,R,R,R,C], each voxel attending to the S keys of its group of (R/g)^3 voxels."""
    if q.ndim != 5 or not q.shape[1] == q.shape[2] == q.shape[3]:
        raise RuntimeError(f"{fn}: q must be [B,R,R,R,C], got {tuple(q.shape)}")
    B, R, C = int(q.shape[0]), int(q.shape[1]), int(q.shape[-1])
    if isinstance(n_group, bool) or not isinstance(n_group, int) or n_group < 1 or R % n_group != 0:
        raise RuntimeError(f"{fn}: n_group must be a positive divisor of R={R}, got {n_group!r}")
    if num_heads < 1 or C % num_heads != 0 or C // num_heads not in (16, 32):
        raise RuntimeError(f"{fn}: need a head dim C/num_heads of 16 or 32, got C={C}, num_heads={num_heads}")
    if (R // n_group) ** 3 * (C // num_heads) > 4096:
        raise RuntimeError(f"{fn}: need (R/n_group)^3 * head dim <= 4096, got R={R}, n_group={n_group}, "
                           f"head dim {C // num_heads}")
    G = B * n_group ** 3
    if k.ndim != 3 or k.shape[0] != G or k.shape[2] != C or not 1 <= k.shape[1] <= 4096 or v.shape != k.shape:
        raise RuntimeError(f"{fn}: k and v must be [{G}, S, {C}] with 1 <= S <= 4096, got {tuple(k.shape)} and "
                           f"{tuple(v.shape)}")
    _check_cuda_float(fn, [("q", q), ("k", k), ("v", v)])
    return _GroupAttn.apply(q, k, v, n_group, num_heads)


class CrossAttention(nn.Module):
    """The parameters of LaRa's ``nn.MultiheadAttention(inner_dim, num_heads, kdim=vdim=cond_dim, bias=False,
    batch_first=True)`` under its names and initialisation: ``q_proj_weight``, ``k_proj_weight``, ``v_proj_weight``
    and ``out_proj.weight``."""

    def __init__(self, embed_dim: int, num_heads: int, cond_dim: int):
        super().__init__()
        self.embed_dim, self.num_heads = embed_dim, num_heads
        self.q_proj_weight = nn.Parameter(torch.empty(embed_dim, embed_dim))
        self.k_proj_weight = nn.Parameter(torch.empty(embed_dim, cond_dim))
        self.v_proj_weight = nn.Parameter(torch.empty(embed_dim, cond_dim))
        self.out_proj = nn.Linear(embed_dim, embed_dim, bias=False)
        for w in (self.q_proj_weight, self.k_proj_weight, self.v_proj_weight):
            nn.init.xavier_uniform_(w)


class GroupAttBlock(nn.Module):
    """LaRa's ``GroupAttBlock`` (network.py:57-102) with LaRa's constructor and parameter names; ``eps`` is unused, as
    in LaRa (its LayerNorms take the default 1e-5)."""

    def __init__(self, inner_dim: int, cond_dim: int, num_heads: int, eps: float = 1e-6, mlp_ratio: float = 2.):
        super().__init__()
        if inner_dim % 32 != 0 or not 32 <= inner_dim <= 512:
            raise ValueError(f"GroupAttBlock: inner_dim must be a multiple of 32 up to 512, got {inner_dim}")
        if num_heads < 1 or inner_dim % num_heads != 0 or inner_dim // num_heads not in (16, 32):
            raise ValueError(f"GroupAttBlock: need a head dim inner_dim/num_heads of 16 or 32, got {inner_dim}/"
                             f"{num_heads}")
        if cond_dim == inner_dim or cond_dim < 1:
            raise ValueError(f"GroupAttBlock: cond_dim must be positive and differ from inner_dim, got {cond_dim}")
        self.num_heads = num_heads
        self.norm1 = nn.LayerNorm(inner_dim)
        self.cross_attn = CrossAttention(inner_dim, num_heads, cond_dim)
        self.cnn = nn.Conv3d(inner_dim, inner_dim, kernel_size=3, padding=1, bias=False)
        self.norm2 = nn.LayerNorm(inner_dim)
        self.norm3 = nn.LayerNorm(inner_dim)
        hidden = int(inner_dim * mlp_ratio)
        self.mlp = nn.Sequential(nn.Linear(inner_dim, hidden), nn.GELU(), nn.Dropout(0.0), nn.Linear(hidden, inner_dim),
                                 nn.Dropout(0.0))

    def forward(self, x, cond, group_axis: int, block_size: int):
        """LaRa's signature: x [B,C,D,H,W], cond [B g^3, S, cond_dim] -> [B,C,D,H,W] (channels_last_3d memory)."""
        fn = "GroupAttBlock.forward"
        if not isinstance(x, torch.Tensor) or x.ndim != 5:
            raise RuntimeError(f"{fn}: x must be [B,C,D,H,W]")
        if group_axis * block_size != x.shape[2]:
            raise RuntimeError(f"{fn}: group_axis * block_size must be D={x.shape[2]}, got {group_axis} * {block_size}")
        n3, c = self.forward_cl(x.permute(0, 2, 3, 4, 1), None, cond, group_axis)
        return (n3 + c).permute(0, 4, 1, 2, 3)

    def forward_cl(self, a, b, cond, n_group: int):
        """The channels-last entry: the block's input is ``a + b`` (b None: ``a``), a [B,R,R,R,C]; returns the block's
        output un-added, ``(n3, cnn(n3))``, both [B,R,R,R,C], so the next add fuses into the next LayerNorm."""
        fn = "GroupAttBlock.forward_cl"
        C = self.norm1.normalized_shape[0]
        if not isinstance(a, torch.Tensor) or a.ndim != 5 or not a.shape[1] == a.shape[2] == a.shape[3] or \
                a.shape[4] != C:
            raise RuntimeError(f"{fn}: the volume must be [B,R,R,R,{C}], got "
                               f"{tuple(a.shape) if isinstance(a, torch.Tensor) else type(a)}")
        Cc = self.cross_attn.k_proj_weight.shape[1]
        if not isinstance(cond, torch.Tensor) or cond.ndim != 3 or cond.shape[2] != Cc:
            raise RuntimeError(f"{fn}: cond must be [B g^3, S, {Cc}], got "
                               f"{tuple(cond.shape) if isinstance(cond, torch.Tensor) else type(cond)}")
        if b is None:
            x, n1 = a, add_layer_norm(a, None, self.norm1, fn)
        else:
            x, n1 = add_layer_norm(a, b, self.norm1, fn)
        at = self.cross_attn
        q = F.linear(n1, at.q_proj_weight)
        k = F.linear(cond, at.k_proj_weight)
        v = F.linear(cond, at.v_proj_weight)
        o = group_attention(q, k, v, n_group, self.num_heads, fn)
        y, n2 = add_layer_norm(x, at.out_proj(o), self.norm2, fn)
        _, n3 = add_layer_norm(y, self.mlp(n2), self.norm3, fn)
        c = self.cnn(n3.permute(0, 4, 1, 2, 3)).permute(0, 2, 3, 4, 1)
        return n3, c


class VolTransformer(nn.Module):
    """LaRa's ``VolTransformer`` (network.py:105-164) with LaRa's constructor and parameter names (``pos_embed``,
    ``layers.i.*``, ``norm``, ``deconv``)."""

    def __init__(self, embed_dim: int, image_feat_dim: int, n_groups: list, vol_low_res: int, vol_high_res: int,
                 out_dim: int, num_layers: int, num_heads: int, eps: float = 1e-6):
        super().__init__()
        if any(not isinstance(g, int) or g < 1 or vol_low_res % g != 0 for g in n_groups) or not n_groups:
            raise ValueError(f"VolTransformer: n_groups must be positive divisors of {vol_low_res}, got {n_groups}")
        self.vol_low_res, self.vol_high_res, self.out_dim = vol_low_res, vol_high_res, out_dim
        self.n_groups = list(n_groups)
        self.block_size = [vol_low_res // g for g in n_groups]
        self.embed_dim = embed_dim
        self.pos_embed = nn.Parameter(torch.randn(1, embed_dim, vol_low_res, vol_low_res, vol_low_res) *
                                      (1. / embed_dim) ** 0.5)
        self.layers = nn.ModuleList([GroupAttBlock(embed_dim, image_feat_dim, num_heads, eps)
                                     for _ in range(num_layers)])
        self.norm = nn.LayerNorm(embed_dim, eps=eps)
        self.deconv = nn.ConvTranspose3d(embed_dim, out_dim, kernel_size=2, stride=2, padding=0)

    def forward(self, image_feats):
        """``image_feats``: LaRa's ``[B,V,Cc,D,D,D]`` volume, or the list of condition blocks
        ``[B g^3, V bs_c^3, Cc]``, one per ``n_groups`` entry (``FeatVolume.cond_tokens``) -> x_up
        ``[B,2R,2R,2R,out_dim]``, contiguous."""
        fn = "VolTransformer.forward"
        if isinstance(image_feats, torch.Tensor):
            if image_feats.ndim != 6:
                raise RuntimeError(f"{fn}: image_feats must be [B,V,C,D,D,D], got {tuple(image_feats.shape)}")
            D = image_feats.shape[3]
            if any(D % g != 0 for g in self.n_groups):
                raise RuntimeError(f"{fn}: the volume's size {D} must be a multiple of every n_groups entry")
            conds = [_cond_blocks(image_feats, g) for g in self.n_groups]
            B = int(image_feats.shape[0])
        else:
            conds = list(image_feats)
            if len(conds) != len(self.n_groups):
                raise RuntimeError(f"{fn}: need one condition tensor per n_groups entry ({len(self.n_groups)}), "
                                   f"got {len(conds)}")
            for g, c in zip(self.n_groups, conds):
                if not isinstance(c, torch.Tensor) or c.ndim != 3 or c.shape[0] % g ** 3 != 0:
                    raise RuntimeError(f"{fn}: the condition of n_group {g} must be [B {g}^3, S, C]")
            B = int(conds[0].shape[0]) // self.n_groups[0] ** 3
            if any(int(c.shape[0]) != B * g ** 3 for g, c in zip(self.n_groups, conds)):
                raise RuntimeError(f"{fn}: the conditions disagree on the batch size")
        a = self.pos_embed.permute(0, 2, 3, 4, 1).expand(B, -1, -1, -1, -1).contiguous()
        b = None
        for i, layer in enumerate(self.layers):
            gi = i % len(self.n_groups)
            a, b = layer.forward_cl(a, b, conds[gi], self.n_groups[gi])
        x = add_layer_norm(a, b, self.norm, fn)[1] if b is not None else add_layer_norm(a, None, self.norm, fn)
        x_up = self.deconv(x.permute(0, 4, 1, 2, 3)).permute(0, 2, 3, 4, 1)
        return x_up.contiguous()


def _cond_blocks(image_feats, n_group):
    """VolTransformer.forward's blocks (network.py:145-150): [B,V,C,D,D,D] -> [B g^3, V bs^3, C]."""
    B, V, C, D, _, _ = image_feats.shape
    bs = D // n_group
    blocks = image_feats.unfold(3, bs, bs).unfold(4, bs, bs).unfold(5, bs, bs)
    blocks = blocks.contiguous().view(B, V, C, n_group ** 3, bs ** 3)
    return torch.einsum("bvcgl->bgvlc", blocks).reshape(B * n_group ** 3, bs ** 3 * V, C)


__all__ = ["GroupAttBlock", "VolTransformer", "CrossAttention", "add_layer_norm", "group_attention"]
