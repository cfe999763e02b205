"""LaRa's fine pass over all B scenes of a batch (DESIGN §3.26), the parts that run without a GPU:

* ``FineSubset``'s restatement of ``Network._check_mask`` (lightning/network.py:381-388) is pinned against LaRa's own
  ``_check_mask`` run on the CPU under the same seeds: both branches and neither, ``training`` on and off, and counts on
  either side of the fp32 1e-3 and 0.5 boundaries at P = 524288.  LaRa's masks are recorded in
  tests/golden/reference/test_fine_pass_batch.npz by ``record_reference``:

      python tests/test_fine_pass_batch.py OUT_DIR LARA_CHECKOUT && cp OUT_DIR/test_fine_pass_batch.npz tests/golden/reference/

* ``FineSubset``'s counts, offsets, pairs and rows equal ``nonzero``'s, for empty and full scenes and B = 1;
* every argument check of ``sample_batch_point_feats``, the batch form of ``FineHead.fine_shs`` and the C entries
  ``srf_point_feats_scenes_*`` rejects bad input before any launch.

The GPU side is tests/test_gpu_fine_pass_batch.py.
"""
import ctypes
import os
import sys
import types

import numpy as np
import pytest
import torch

from helpers import fingerprint, reference_record
from lara_b200.multiview import FineSubset

MODULE = "test_fine_pass_batch"
P_LARA = 524288


def _mask_with_count(P, count, seed):
    """A bool mask [P] with exactly `count` True entries at seeded positions."""
    g = torch.Generator().manual_seed(seed)
    m = torch.zeros(P, dtype=torch.bool)
    m[torch.randperm(P, generator=g)[:count]] = True
    return m


# case -> (P, per-scene counts, training, seed of the _check_mask draws)
CHECK_CASES = {
    "branches_training": (4096, (2, 3000, 1000, 0, 4096), True, 11),
    "branches_eval": (4096, (2, 3000, 1000, 0, 4096), False, 12),
    "no_branch": (4096, (1000, 2048, 5), False, 13),
    "no_branch_training": (4096, (1000, 2048, 5), True, 14),
    # fp32(524) / 2^19 = 9.9945e-4 < fp32(1e-3) <= fp32(525) / 2^19; 2^18 / 2^19 = 0.5 is not > 0.5
    "boundary_low": (P_LARA, (524, 525), True, 15),
    "boundary_high": (P_LARA, (262144, 262145), True, 16),
    "boundary_high_eval": (P_LARA, (262144, 262145), False, 17),
}


def _case_masks(name):
    P, counts, training, seed = CHECK_CASES[name]
    return torch.stack([_mask_with_count(P, c, 100 * seed + b) for b, c in enumerate(counts)]), training, seed


def _record(masks):
    return {"count": np.array([int(m.sum()) for m in masks], dtype=np.int64),
            "masks": fingerprint(masks.numpy())}


def record_reference(lara, dev="cpu"):
    """LaRa's own ``Network._check_mask`` on every scene of each case, in scene order, under the case's seed."""
    from test_decoder_layout import _import_reference_network
    net = _import_reference_network(lara)
    out = {}
    for name in CHECK_CASES:
        masks, training, seed = _case_masks(name)
        fake = types.SimpleNamespace(device=torch.device(dev), training=training)
        torch.manual_seed(seed)
        checked = torch.stack([net.Network._check_mask(fake, m) for m in masks])
        out[name] = _record(checked)
    return out


@pytest.mark.parametrize("name", list(CHECK_CASES))
def test_check_mask_matches_lara(name):
    ref = reference_record(MODULE, name)
    masks, training, seed = _case_masks(name)
    torch.manual_seed(seed)
    sub = FineSubset(masks, check=True, training=training)
    got = _record(sub.masks)
    assert np.array_equal(got["count"], ref["count"]), (got["count"], ref["count"])
    assert got["masks"] == ref["masks"]
    assert sub.counts == [int(c) for c in ref["count"]]


def test_check_mask_draws_only_where_lara_draws():
    """No branch: the masks are kept as they are and the RNG is not advanced; a branch draws one rand per scene."""
    masks, _, _ = _case_masks("no_branch")
    torch.manual_seed(3)
    sub = FineSubset(masks, check=True, training=True)
    assert sub.masks is masks
    after = torch.rand(1)
    torch.manual_seed(3)
    assert torch.equal(after, torch.rand(1))


def test_check_mask_ratio_is_fp32():
    """The ratio is fp32(count) / fp32(P) compared with fp32 thresholds, as torch computes it."""
    for P, c in ((P_LARA, 524), (P_LARA, 525), (P_LARA, 262144), (P_LARA, 262145), (1000, 1), (3, 2)):
        r = torch.tensor(c) / np.prod((P,))
        assert r.dtype == torch.float32
        assert bool(r < 1e-3) == bool(np.float32(c) / np.float32(P) < np.float32(1e-3))
        assert bool(r > 0.5) == bool(np.float32(c) / np.float32(P) > np.float32(0.5))


@pytest.mark.parametrize("counts", [(5, 0, 64, 17), (64, 64), (0, 0, 0), (9,), (0,), (64,)])
def test_subset_layout_equals_nonzero(counts):
    P = 64
    masks = torch.stack([_mask_with_count(P, c, 7 + b) for b, c in enumerate(counts)])
    sub = FineSubset(masks)
    nz = masks.nonzero()
    assert sub.counts == list(counts) and sub.n == sum(counts)
    assert sub.offsets == [0] + list(np.cumsum(counts))
    assert torch.equal(sub.nz, nz) and torch.equal(sub.idx, nz[:, 1])
    assert sub.rows.dtype == torch.int32 and torch.equal(sub.rows.long(), nz[:, 0] * P + nz[:, 1])
    if len(counts) == 1:
        assert sub.offsets_d is None
    else:
        assert sub.offsets_d.tolist() == sub.offsets


def test_subset_rejects_bad_masks():
    with pytest.raises(RuntimeError, match="bool tensor"):
        FineSubset(torch.zeros(2, 8))
    with pytest.raises(RuntimeError, match="bool tensor"):
        FineSubset(torch.zeros(8, dtype=torch.bool))
    with pytest.raises(RuntimeError, match="at least one scene"):
        FineSubset(torch.zeros(0, 8, dtype=torch.bool))
    big = torch.zeros(2 ** 31 // 2 ** 20 * 2, 1, dtype=torch.bool).expand(-1, 2 ** 20)     # B*P = 2^32, no storage
    with pytest.raises(RuntimeError, match="int32 index range"):
        FineSubset(big)


# ---- argument checks of the Python entries --------------------------------------------------------------------------
def _batch_inputs(B=2, Vs=2, V=3, P=16, H=8, W=8, dtype=torch.float32):
    masks = torch.zeros(B, P, dtype=torch.bool)
    masks[:, ::3] = True
    sub = FineSubset(masks)
    centers = torch.rand(B, P, 3, dtype=dtype)
    img_ref = torch.rand(B, Vs, 3, H, W, dtype=dtype)
    rend = {"image": torch.rand(B, V, H, W, 3, dtype=dtype), "acc_map": torch.rand(B, V, H, W, dtype=dtype),
            "depth": torch.rand(B, V, H, W, 1, dtype=dtype)}
    return sub, centers, img_ref, rend, torch.rand(B, Vs, 4, 4, dtype=dtype), torch.rand(B, Vs, 3, 3, dtype=dtype)


@pytest.mark.parametrize("what", ["subset", "centers", "img_ref", "image", "image_views", "acc_map", "depth", "w2cs",
                                  "ixts"])
def test_sample_batch_point_feats_rejects_bad_shapes(what):
    from lara_b200.point_feats import sample_batch_point_feats
    sub, centers, img_ref, rend, w2c, ixt = _batch_inputs()
    bad = {"subset": lambda: (sub.masks, centers, img_ref, rend, w2c, ixt),
           "centers": lambda: (sub, centers[:, :-1], img_ref, rend, w2c, ixt),
           "img_ref": lambda: (sub, centers, img_ref[:, :, :2], rend, w2c, ixt),
           "image": lambda: (sub, centers, img_ref, {**rend, "image": rend["image"][..., :2]}, w2c, ixt),
           "image_views": lambda: (sub, centers, img_ref, {**rend, "image": rend["image"][:, :1]}, w2c, ixt),
           "acc_map": lambda: (sub, centers, img_ref, {**rend, "acc_map": rend["acc_map"][:, :2]}, w2c, ixt),
           "depth": lambda: (sub, centers, img_ref, {**rend, "depth": rend["depth"][..., 0]}, w2c, ixt),
           "w2cs": lambda: (sub, centers, img_ref, rend, w2c[:, :1], ixt),
           "ixts": lambda: (sub, centers, img_ref, rend, w2c, ixt[:1])}[what]()
    with pytest.raises((RuntimeError, TypeError), match="sample_batch_point_feats"):
        sample_batch_point_feats(*bad)


def test_sample_batch_point_feats_rejects_dtype_device_and_constants_requiring_grad():
    from lara_b200.point_feats import sample_batch_point_feats
    with pytest.raises(RuntimeError, match="Float"):
        sample_batch_point_feats(*_batch_inputs(dtype=torch.float64))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        sample_batch_point_feats(*_batch_inputs())
    with pytest.raises(KeyError):
        sub, centers, img_ref, rend, w2c, ixt = _batch_inputs()
        sample_batch_point_feats(sub, centers, img_ref, {"image": rend["image"], "depth": rend["depth"]}, w2c, ixt)
    for k in range(3):
        sub, centers, img_ref, rend, w2c, ixt = _batch_inputs()
        consts = [img_ref, w2c, ixt]
        consts[k] = consts[k].clone().requires_grad_(True)
        with pytest.raises(RuntimeError, match="requires grad"):
            sample_batch_point_feats(sub, centers, consts[0], rend, consts[1], consts[2])


def test_fine_shs_batch_rejects_bad_arguments():
    from lara_b200.fine_head import FineHead
    head = FineHead(16, 12)
    B, N, K, Vs = 2, 8, 2, 3
    masks = torch.zeros(B, N * K, dtype=torch.bool)
    masks[:, 1::3] = True
    sub = FineSubset(masks)
    vf, pf, shs = torch.rand(B, N, 16), torch.rand(Vs, 8, sub.n), torch.rand(B, N * K, 4, 3)
    fn = "FineHead.fine_shs"
    cases = [(torch.rand(B, N, 8), K, sub, pf, shs),                 # D
             (vf, K, masks[:, :-1], pf, shs),                         # masks shape
             (vf, K, masks.float(), pf, shs),                         # masks dtype
             (vf, K, "masks", pf, shs),                               # neither masks nor subset
             (vf, K, FineSubset(masks[:1]), pf, shs),                 # subset of another batch
             (vf, K, sub, pf, shs[:, :-1]),                           # shs_coarse
             (vf, K, sub, pf[:, :4], shs),                            # point_feats channels
             (vf, K, sub, pf[:, :, :-1], shs),                        # point_feats count
             (vf, K, sub, pf.double(), shs)]                          # dtype
    for args in cases:
        with pytest.raises(RuntimeError, match=fn):
            head.fine_shs(*args)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        head.fine_shs(vf, K, sub, pf, shs)
    with pytest.raises(RuntimeError, match="K must be"):
        head.fine_shs(vf, 0, sub, pf, shs)


# ---- the C entries --------------------------------------------------------------------------------------------------
def _offsets(*v):
    return (ctypes.c_int64 * len(v))(*v)


def test_point_feats_scenes_c_entries_reject_bad_arguments_before_any_launch(lib):
    from lara_b200 import _lib
    Pp = ctypes.c_void_p(256)           # never dereferenced: the checks come before any CUDA call
    addr = _lib.PfImageAddr(0, 3 * 64, 64, 8, 1)
    ref = ctypes.byref(addr)

    def fwd(S=2, Vs=2, Vr=2, P=4, n=5, H=8, W=8, off=None, rows=Pp, ins=None, a=ref, feats=Pp):
        off = _offsets(0, 2, 5) if off is None else off
        ins = [Pp] * 4 if ins is None else ins        # centers, w2cs, ixts, img_ref
        return lib.srf_point_feats_scenes_forward(None, S, Vs, Vr, P, n, H, W, off, rows, *ins, a, Pp, Pp, Pp, feats)

    def bwd(S=2, Vs=2, Vr=2, P=4, n=5, H=8, W=8, off=None, rows=Pp, g=Pp, ws=None):
        off = _offsets(0, 2, 5) if off is None else off
        return lib.srf_point_feats_scenes_backward(None, S, Vs, Vr, P, n, H, W, off, rows, Pp, Pp, Pp, Pp, ref, Pp, Pp,
                                                   Pp, g, Pp, Pp, Pp, Pp, ws)

    def err():
        return lib.srf_last_error()

    for kw, msg in ((dict(S=0), b"scenes"), (dict(S=129, off=_offsets(*range(130))), b"scenes"),
                    (dict(Vs=0), b"bad sizes"), (dict(Vr=1), b"bad sizes"), (dict(n=-1), b"bad sizes"),
                    (dict(H=0), b"bad sizes"), (dict(W=0), b"bad sizes"), (dict(P=-1), b"bad sizes"),
                    (dict(P=2 ** 30), b"int32 index range"),
                    (dict(Vr=40000, Vs=2), b"65535"),
                    (dict(off=_offsets(1, 2, 5)), b"offsets must run from 0 to n"),
                    (dict(off=_offsets(0, 2, 4)), b"offsets must run from 0 to n"),
                    (dict(off=_offsets(0, 3, 2, 5), S=3), b"must not decrease"),
                    (dict(off=_offsets(0, 0, 5)), b"at most P"),
                    (dict(off=_offsets(0, 4, 9), rows=None, n=9, P=4), b"at most P")):
        assert fwd(**kw) != 0, kw
        assert msg in err(), (kw, err())
        assert b"srf_point_feats_scenes_forward" in err()
    assert bwd(S=0) != 0 and b"srf_point_feats_scenes_backward" in err()
    assert bwd(S=3, off=_offsets(0, 3, 2, 5)) != 0 and b"must not decrease" in err()
    for k in range(4):
        ins = [Pp] * 4
        ins[k] = None
        assert fwd(ins=ins) != 0 and b"null input pointer" in err()
    assert fwd(off=ctypes.c_void_p(0)) != 0 and b"null host offsets" in err()
    assert fwd(a=None) != 0 and b"null host offsets or img_ref strides" in err()
    assert fwd(feats=None) != 0 and b"null output pointer" in err()
    assert bwd(g=None) != 0 and b"null upstream gradient" in err()
    assert bwd(ws=8) != 0 and b"workspace must be 256-byte aligned" in err()
    # n == 0: nothing to read, the forward launches nothing
    assert fwd(n=0, off=_offsets(0, 0, 0), ins=[None, Pp, Pp, Pp], feats=None) == 0
    # the deterministic workspace query
    b = ctypes.c_size_t()
    assert lib.srf_point_feats_scenes_deterministic_workspace_bytes(3, 4, 16, 16, ctypes.byref(b)) == 0
    assert b.value >= 5 * 3 * 4 * 16 * 16 * 8
    one = ctypes.c_size_t()
    assert lib.srf_point_feats_deterministic_workspace_bytes(4, 16, 16, ctypes.byref(one)) == 0
    assert lib.srf_point_feats_scenes_deterministic_workspace_bytes(1, 4, 16, 16, ctypes.byref(b)) == 0
    assert b.value == one.value
    for args in ((0, 4, 16, 16), (129, 4, 16, 16), (1, 0, 16, 16), (1, 4, 0, 16)):
        assert lib.srf_point_feats_scenes_deterministic_workspace_bytes(*args, ctypes.byref(b)) != 0


if __name__ == "__main__":
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_reference_records import save
    os.makedirs(sys.argv[1], exist_ok=True)
    save(sys.argv[1], MODULE, record_reference(sys.argv[2], "cpu"))
