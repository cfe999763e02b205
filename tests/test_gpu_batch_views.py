"""B scenes in one launch set (``render_batch_views`` / ``render_batch_subset_views``, DESIGN §3.21) against the per-scene
calls they replace (``render_scene_views`` / ``render_subset_views`` of each scene alone): outputs, radii and
``n_contrib`` bit for bit, gradients bit for bit under ``torch.use_deterministic_algorithms(True)`` and within the
atomics' rounding otherwise, ragged subsets with an empty and a full mask, the stage-2 re-run after an overflow, and
B = 1."""
import warnings

import pytest
import torch

from lara_b200 import rasterizer as R
from lara_b200 import scene as S
from lara_b200.debug import unpack_state
from lara_b200.multiview import (OUT_KEYS, render_batch_subset_views, render_batch_views, render_scene_views,
                                 render_subset_views)
from test_chain_per_element import lara_rays

pytestmark = pytest.mark.gpu

H = W = 512


def _batch(B, V, P, seed, dev, big=False):
    """B LaRa-like scenes (raw network outputs) with their own field of view and background, V cameras each, LaRa's
    rays, and fine SH coefficients for every Gaussian."""
    params, settings, rays, shs_fine = [], [], [], []
    for b in range(B):
        sc = S.scene(P, seed + 17 * b, 1)
        s = sc["scales"] * (12.0 if big else 1.0)
        params.append((sc["means3D"], sc["shs"], torch.logit(sc["opacities"]), torch.log(s), sc["rotations"] * 1.7))
        cams = S.cameras(V, H, W, seed + b, fov=0.65 + 0.1 * b)
        bg = torch.tensor([0.2 * b, 0.5, 1.0 - 0.3 * b])
        settings.append([S.settings_for(c, bg, 1, dev, R.GaussianRasterizationSettings) for c in cams])
        rays.append(torch.stack([lara_rays(c) for c in cams]))
        g = torch.Generator().manual_seed(seed + 5 + b)
        shs_fine.append(torch.randn(sc["shs"].shape, generator=g) * 0.6)
    stacked = [torch.stack([p[k] for p in params]).to(dev).contiguous() for k in range(5)]
    return stacked, settings, torch.stack(rays).to(dev).contiguous(), torch.stack(shs_fine).to(dev)


def _leaves(params, grad):
    return [p.detach().clone().requires_grad_(grad) for p in params]


def _weights(out, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return {k: torch.randn(out[k].shape, generator=g, device="cuda") for k in OUT_KEYS}


def _loss(out, w, b=None):
    return sum((out[k] * (w[k] if b is None else w[k][b])).sum() for k in OUT_KEYS)


@pytest.mark.parametrize("P,V", [(131072, 4), (131072, 8), (524288, 8)])
@pytest.mark.parametrize("with_rays", [True, False])
def test_forward_bit_for_bit(cuda_device, P, V, with_rays):
    B = 3
    params, settings, rays, _ = _batch(B, V, P, 3, cuda_device)
    rr = rays if with_rays else None
    leaves = _leaves(params, True)
    out = render_batch_views(*leaves, settings, rays=rr, raw_activations=True, keep_binning=True)
    st = out["binning"].state
    keys = (OUT_KEYS if with_rays else ("image",)) + ("radii",)
    for b in range(B):
        one = [t[b] for t in _leaves(params, True)]
        ref = render_scene_views(*one, settings[b], rays=rr[b] if with_rays else None, raw_activations=True,
                                 keep_binning=True)
        for k in keys:
            assert torch.equal(out[k][b], ref[k]), (b, k)
        rst = ref["binning"].state
        for j in range(V):
            a, r = unpack_state(st, P, H, W, b * V + j), unpack_state(rst, P, H, W, j)
            assert torch.equal(a["n_contrib"], r["n_contrib"]), (b, j)
            assert torch.equal(a["ranges"], r["ranges"]), (b, j)


def test_forward_only_bit_for_bit(cuda_device):
    B, V, P = 3, 4, 131072
    params, settings, rays, _ = _batch(B, V, P, 4, cuda_device)
    with torch.no_grad():
        out = render_batch_views(*params, settings, rays=rays, raw_activations=True)
        assert not out["image"].requires_grad
        for b in range(B):
            ref = render_scene_views(*[t[b] for t in params], settings[b], rays=rays[b], raw_activations=True)
            for k in OUT_KEYS + ("radii",):
                assert torch.equal(out[k][b], ref[k]), (b, k)


def _grads(params, settings, rays, seed, batched):
    B = len(settings)
    leaves = _leaves(params, True)
    if batched:
        out = render_batch_views(*leaves, settings, rays=rays, raw_activations=True)
        _loss(out, _weights(out, seed)).backward()
        return [[t.grad[b] for t in leaves] for b in range(B)]
    w = None
    res = []
    for b in range(B):
        one = [t[b].detach().clone().requires_grad_(True) for t in params]
        out = render_scene_views(*one, settings[b], rays=rays[b], raw_activations=True)
        if w is None:
            shapes = {k: (B,) + tuple(out[k].shape) for k in OUT_KEYS}
            g = torch.Generator(device="cuda").manual_seed(seed)
            w = {k: torch.randn(shapes[k], generator=g, device="cuda") for k in OUT_KEYS}
        _loss(out, w, b).backward()
        res.append([t.grad for t in one])
    return res


@pytest.mark.parametrize("P,V", [(131072, 4), (524288, 8)])
def test_backward(cuda_device, P, V):
    params, settings, rays, _ = _batch(3, V, P, 5, cuda_device)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        gb = _grads(params, settings, rays, 9, True)
        gs = _grads(params, settings, rays, 9, False)
    finally:
        torch.use_deterministic_algorithms(prev)
    for b in range(3):
        for k, (a, r) in enumerate(zip(gb[b], gs[b])):
            assert torch.equal(a, r), (b, k)
    gb = _grads(params, settings, rays, 9, True)
    for b in range(3):
        for k, (a, r) in enumerate(zip(gb[b], gs[b])):
            assert torch.allclose(a, r, rtol=1e-3, atol=1e-5 * float(r.abs().max()) + 1e-9), (b, k)


def test_subset_ragged(cuda_device):
    B, V, P = 3, 4, 131072
    params, settings, rays, shs_full = _batch(B, V, P, 6, cuda_device)
    g = torch.Generator(device="cuda").manual_seed(1)
    masks = torch.stack([torch.rand(P, generator=g, device="cuda") < 0.5,
                         torch.zeros(P, dtype=torch.bool, device="cuda"),
                         torch.ones(P, dtype=torch.bool, device="cuda")])
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        leaves = _leaves(params, True)
        fine = torch.cat([shs_full[b][masks[b]] for b in range(B)]).requires_grad_(True)
        coarse = render_batch_views(*leaves, settings, rays=rays, raw_activations=True, keep_binning=True)
        out = render_batch_subset_views(coarse["binning"], masks, fine)
        w = _weights({k: out[k + "_fine"] for k in OUT_KEYS}, 11)
        sum((out[k + "_fine"] * w[k]).sum() for k in OUT_KEYS).backward()
        n0 = 0
        for b in range(B):
            one = [t[b].detach().clone().requires_grad_(True) for t in params]
            fb = shs_full[b][masks[b]].clone().requires_grad_(True)
            cb = render_scene_views(*one, settings[b], rays=rays[b], raw_activations=True, keep_binning=True)
            ref = render_subset_views(cb["binning"], masks[b], fb)
            for k in OUT_KEYS:
                assert torch.equal(out[k + "_fine"][b], ref[k + "_fine"]), (b, k)
            assert torch.equal(out["radii_fine"][b], ref["radii_fine"]), b
            if fb.shape[0]:
                sum((ref[k + "_fine"] * w[k][b]).sum() for k in OUT_KEYS).backward()
                assert torch.equal(fine.grad[n0:n0 + fb.shape[0]], fb.grad), b
                for k, t in enumerate(one):
                    if k != 1:
                        assert torch.equal(leaves[k].grad[b], t.grad), (b, k)
            else:
                for k in (0, 2, 3, 4):
                    assert not leaves[k].grad[b].any(), (b, k)
            n0 += fb.shape[0]
    finally:
        torch.use_deterministic_algorithms(prev)


def test_overflow_rerun(cuda_device, monkeypatch):
    B, V, P = 3, 4, 131072
    params, settings, rays, _ = _batch(B, V, P, 7, cuda_device, big=True)
    # a fresh capacity guess, which these large splats overflow; the suite's own guess comes back after the test
    monkeypatch.setattr(R, "_capacity_hwm", {})
    # the counts are read inside the forward, so the re-run happens before the epilogue reads the images
    monkeypatch.setenv("SRF_SYNC_NUM_RENDERED", "1")
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)
        out = render_batch_views(*_leaves(params, True), settings, rays=rays, raw_activations=True, keep_binning=True)
    counts = out["binning"].state.resolve()
    monkeypatch.delenv("SRF_SYNC_NUM_RENDERED")
    assert max(counts) > 8 * P, "the case must overflow the first capacity guess"
    for b in range(B):
        ref = render_scene_views(*[t[b] for t in _leaves(params, True)], settings[b], rays=rays[b], raw_activations=True)
        for k in OUT_KEYS + ("radii",):
            assert torch.equal(out[k][b], ref[k]), (b, k)


def test_single_scene(cuda_device):
    params, settings, rays, _ = _batch(1, 4, 131072, 8, cuda_device)
    out = render_batch_views(*_leaves(params, True), settings, rays=rays, raw_activations=True)
    ref = render_scene_views(*[t[0] for t in _leaves(params, True)], settings[0], rays=rays[0], raw_activations=True)
    for k in OUT_KEYS + ("radii",):
        assert torch.equal(out[k][0], ref[k]), k
