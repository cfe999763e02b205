"""LaRa's training batch on the GPU (lara_b200.batch.assemble_batch, srf_batch_assemble) on an H100.

* On the record's raw inputs the kernel equals LaRa's record (tests/golden/reference/test_batch*.npz) under the rules
  of DESIGN §3.23: colour and mask bit for bit, rays bit for bit where their fp64 sum is exact and within one fp32 ulp
  elsewhere, normals within 2 * 2^-24 * sum_j |n_j R_ij| of the exact product.
* At LaRa's size (B = 3, N = 8, 512², seeded synthetic views) it equals test_batch's torch CPU restatement bit for bit
  on every output, with and without normals; the normals are also checked against the bound.
* Pinned host, pageable host and device inputs give the same bits, at a size whose rows are not 16-byte multiples;
  repeats are bit-identical; two batches issued back to back without a synchronise both come out right.
"""
from __future__ import annotations

import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from helpers import reference_record  # noqa: E402
from test_batch import (CASES, U, Cfg, assemble_reference, check_against, collate, dataset_samples,  # noqa: E402
                        normal_bound, seed_all, synthetic_metas)

pytestmark = pytest.mark.gpu

OUTPUTS = ("tar_rgb", "tar_msk", "tar_nrm", "tar_rays", "tar_rays_down")


def views_raw(seed, B, H, W, split="train", n_group=4, normals=True):
    """A collated raw batch of B scenes from GobjverseViews on seeded synthetic contents (host, pageable)."""
    from lara_b200.batch import GobjverseViews
    ds = GobjverseViews(Cfg(split, n_group, H, W, normals), metas=synthetic_metas(seed, H, W, n_scenes=B + 1))
    seed_all(seed)
    return collate([ds[i] for i in range(B)])


def pinned(raw):
    return {k: (v.pin_memory() if isinstance(v, torch.Tensor) else v) for k, v in raw.items()}


def on_device(raw, dev):
    return {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in raw.items()}


def assert_same(out, ref, keys=OUTPUTS):
    for k in keys:
        if k not in ref:
            assert k not in out, k
            continue
        a, b = out[k].cpu(), ref[k].cpu()
        assert a.dtype == b.dtype and a.shape == b.shape, k
        assert torch.equal(a, b), f"{k}: {(a != b).sum().item()} elements differ"


@pytest.mark.parametrize("case", list(CASES))
def test_kernel_equals_lara_record(case, cuda_device):
    from lara_b200.batch import assemble_batch
    for j, s in enumerate(dataset_samples(case)):
        raw = collate([s])
        out = assemble_batch(raw, cuda_device)
        torch.cuda.synchronize()
        n = check_against(out, raw, reference_record("test_batch", f"{case}_{j}"))
        print(f"{case}_{j}: {n} ray components with an inexact fp64 sum")


@pytest.mark.parametrize("normals", [True, False], ids=["normals", "no_normals"])
def test_lara_size_equals_restatement(normals, cuda_device):
    from lara_b200.batch import assemble_batch
    raw = views_raw(21, 3, 512, 512, normals=normals)
    assert tuple(raw["tar_rgba"].shape) == (3, 8, 512, 512, 4)
    out = assemble_batch(pinned(raw), cuda_device)
    ref = assemble_reference(raw, with_exact=True)
    assert_same(out, ref)
    assert tuple(out["tar_rays_down"].shape) == (3, 8, 32, 32, 6)
    if normals:
        assert tuple(out["tar_nrm"].shape) == (3, 512, 8 * 512, 3)
        exact, mag = normal_bound(raw)
        assert bool(((out["tar_nrm"].cpu().double() - exact).abs() <= 2 * U * mag).all())
    ex = ref["exact"]
    print(f"{int(ex.numel() - ex.sum())} of {ex.numel()} ray components with an inexact fp64 sum")
    # the small tensors come along, moved
    for k in ("tar_c2w", "tar_w2c", "tar_ixt", "near_far", "bg_color", "i2w"):
        assert out[k].is_cuda and torch.equal(out[k].cpu(), raw[k])
    assert out["meta"] is raw["meta"]


def test_sources_repeats_and_odd_rows(cuda_device):
    """H = 33, W = 45: a row of rgb is 540 B and of rays 1080 B, so the 128-bit stores start at every alignment."""
    from lara_b200.batch import assemble_batch
    raw = views_raw(5, 2, 33, 45)
    ref = assemble_reference(raw)
    outs = [assemble_batch(r, cuda_device) for r in (pinned(raw), raw, on_device(raw, cuda_device))]
    outs.append(assemble_batch(on_device(raw, cuda_device)))       # device taken from the batch
    torch.cuda.synchronize()
    for o in outs:
        assert_same(o, ref)
    assert tuple(outs[0]["tar_rays_down"].shape) == (2, 8, 2, 2, 6)


def test_back_to_back_without_synchronise(cuda_device):
    from lara_b200.batch import assemble_batch
    raws = [views_raw(s, 3, 256, 256) for s in (31, 32)]
    refs = [assemble_reference(r) for r in raws]
    torch.cuda.synchronize()
    outs = []
    for r in raws:
        p = pinned(r)
        outs.append(assemble_batch(p, cuda_device))
        del p
    torch.cuda.synchronize()
    for o, ref in zip(outs, refs):
        assert_same(o, ref)
    assert not torch.equal(outs[0]["tar_rgb"].cpu(), outs[1]["tar_rgb"].cpu())


def test_test_split_batch_without_normals(cuda_device):
    """LaRa's inference config (load_normal False) on the test split: no tar_nrm, the rest as the restatement."""
    from lara_b200.batch import assemble_batch
    raw = views_raw(9, 1, 64, 96, split="test", normals=False)
    out = assemble_batch(raw, cuda_device)
    assert "tar_nrm" not in out
    assert_same(out, assemble_reference(raw))
    assert bool((raw["bg_color"] == 1).all())
