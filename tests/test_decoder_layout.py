"""Decoder epilogue (next-row, SURVEY 8f rank 4): MLP output -> contiguous Gaussian-parameter tensors.

* CPU: the torch restatement is pinned bit-exactly against the reference's own ``Decoder.forward_coarse`` +
  ``Network.get_offseted_pt`` (lightning/network.py), imported with stub modules for timm / pytorch_lightning and an
  identity MLP; its outputs are recorded in tests/golden/reference/test_decoder_layout.npz (record_reference).
* GPU: the fused kernel vs the restatement -- forward values bit-exact except the sigmoid path (<= 2 ulp), backward
  to 1e-6."""
import sys
import types

import pytest
import torch

from helpers import fingerprint, reference_record, rel_err


def _import_reference_network(lara):
    stubs = {}

    def stub(name, **attrs):
        m = types.ModuleType(name)
        for k, v in attrs.items():
            setattr(m, k, v)
        stubs[name] = m
        return m
    stub("timm")
    stub("pytorch_lightning", LightningModule=torch.nn.Module)
    tv = stub("torchvision")
    tv.transforms = stub("torchvision.transforms")
    saved = {k: sys.modules.get(k) for k in stubs}
    sys.modules.update({k: v for k, v in stubs.items() if k not in sys.modules or k in ("timm", "pytorch_lightning")})
    sys.path.insert(0, lara)
    try:
        import importlib
        for k in [k for k in sys.modules if k == "lightning" or k.startswith("lightning.")]:
            del sys.modules[k]
        net = importlib.import_module("lightning.network")
    finally:
        sys.path.remove(lara)
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
        for k in [k for k in sys.modules if k == "lightning" or k.startswith("lightning.") or k == "tools" or k.startswith("tools.")]:
            del sys.modules[k]
    return net


B, N, K, SH_DIM = 2, 27, 2, 12


def _cpu_inputs():
    g = torch.Generator().manual_seed(0)
    feats = torch.randn((B, N, K * (10 + SH_DIM)), generator=g)
    return feats, torch.rand((1, N, 3), generator=g) - 0.5


def record_reference(lara, dev):
    """LaRa's own decoder layout on the CPU (tests/golden/make_reference_records.py)."""
    net = _import_reference_network(lara)
    sh_dim = SH_DIM
    feats, centers_grid = _cpu_inputs()
    dec = net.Decoder.__new__(net.Decoder)
    torch.nn.Module.__init__(dec)
    dec.K, dec.sh_dim, dec.opacity_dim, dec.scaling_dim, dec.rotation_dim = K, sh_dim, 1, 2, 4
    dec.mlp_coarse = torch.nn.Identity()
    opacity_shift, scaling_shift = -2.1792, -4.2
    ref = dec.forward_coarse(feats, opacity_shift, scaling_shift)        # offset, sh, scaling, rotation, opacity
    fake_self = types.SimpleNamespace(scene_size=1.0, n_offset_groups=16, group_centers=centers_grid)
    ref_centers = net.Network.get_offseted_pt(fake_self, ref[0], K)
    return {"layout": {str(i): fingerprint(t.detach().numpy()) for i, t in enumerate([ref_centers] + list(ref[1:]))}}


def test_decoder_restatement_matches_reference_on_cpu():
    from oracle.torch_restatements import decoder_layout_torch
    feats, centers_grid = _cpu_inputs()
    mine = decoder_layout_torch(feats, centers_grid, K, SH_DIM, -2.1792, -4.2, 0.5 * 1.0 / 16)
    ref = reference_record("test_decoder_layout", "layout")
    assert len(ref) == len(mine)
    for i, t in enumerate(mine):        # centers, sh, scaling, rotation, opacity: values and shape, bit for bit
        assert fingerprint(t.numpy()) == ref[str(i)], i


@pytest.mark.gpu
@pytest.mark.parametrize("B,N,K,sh_dim", [(1, 1000, 2, 12), (3, 4097, 1, 12), (2, 515, 2, 48), (1, 200, 3, 3)])
def test_decoder_layout_kernel_matches_restatement(cuda_device, B, N, K, sh_dim):
    from lara_b200.decoder_layout import gaussians_from_decoder
    from oracle.torch_restatements import decoder_layout_torch
    dev = cuda_device
    g = torch.Generator().manual_seed(N)
    C = 10 + sh_dim
    feats = (torch.randn((B, N, K * C), generator=g) * 2).to(dev)
    grid = (torch.rand((N, 3), generator=g) - 0.5).to(dev)
    ups = None
    res = []
    for fn in (gaussians_from_decoder, decoder_layout_torch):
        x = feats.clone().requires_grad_(True)
        out = fn(x, grid, K, sh_dim, -2.1792, -4.2, 0.03125)
        if ups is None:
            ups = [torch.randn(o.shape, generator=g).to(dev) for o in out]
        torch.autograd.backward(out, ups)
        res.append(([o.detach() for o in out], x.grad.detach()))
    (o1, g1), (o2, g2) = res
    for k, (a, b) in enumerate(zip(o1, o2)):
        assert a.shape == b.shape and a.is_contiguous(), k
        if k == 0:
            assert rel_err(a.cpu().numpy(), b.cpu().numpy()) < 1e-6       # sigmoid: torch's CUDA kernel vs expf-based, <= 2 ulp
        else:
            assert torch.equal(a, b), k
    assert rel_err(g1.cpu().numpy(), g2.cpu().numpy()) < 1e-6
