"""LaRa's training batch on the GPU (lara_b200.batch), CPU side.

* ``GobjverseViews`` picks LaRa's views and backgrounds under the same seeds and gives LaRa's cameras, ``i2w`` and
  ``i2w_down`` bit for bit: LaRa's own ``gobjverse.__getitem__`` ran on seeded synthetic h5 contents and is recorded in
  tests/golden/reference/test_batch*.npz (``record_reference``; ``python tests/test_batch.py OUT_DIR LARA_CHECKOUT``
  writes OUT_DIR/test_batch*.npz with tests/golden/make_reference_records.py's writer).
* ``assemble_reference``, a torch CPU restatement of ``srf_batch_assemble`` (fp32 colour and normal decode, fp64 rays
  and rotation), equals that record under the rules of DESIGN §3.23: colour and mask bit for bit, rays bit for bit
  where their fp64 three-term sum is exact and within one fp32 ulp elsewhere, normals within
  2 * 2^-24 * sum_j |n_j R_ij| of the exact product.  LaRa's own fp32 BLAS product is held to the general three-term
  bound gamma_3 = 3 * 2^-24 / (1 - 3 * 2^-24) instead: the record exceeds 2 * 2^-24 in a few values.
* The C entry rejects bad arguments before any launch; the Python layer rejects inputs that are not uint8.
"""
from __future__ import annotations

import importlib
import os
import random
import sys
import types

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from helpers import reference_record  # noqa: E402

U = 2.0 ** -24          # fp32 unit roundoff


# ---- seeded synthetic h5 contents ----

def synthetic_metas(seed, H, W, n_scenes=12, n_views=12):
    """A mapping with the keys of LaRa's gobjaverse.h5: per scene ``groups/groups_{4,2}_i`` view lists, ``c2w_v``,
    ``fov_v`` and uint8 ``image_v`` (alpha 0, 255 and values between) and ``normal_v``."""
    rng = np.random.default_rng(seed)
    metas = {}
    for s in range(n_scenes):
        perm = rng.permutation(n_views)
        groups = {f"groups_4_{i}": perm[i::4].copy() for i in range(4)}
        groups.update({f"groups_2_{i}": perm[i::2].copy() for i in range(2)})
        scene = {"groups": groups}
        for v in range(n_views):
            q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
            c2w = np.eye(4, dtype=np.float32)
            c2w[:3, :3] = q
            d = rng.standard_normal(3)
            c2w[:3, 3] = d / np.linalg.norm(d) * rng.uniform(1.5, 2.5)
            scene[f"c2w_{v}"] = c2w
            scene[f"fov_{v}"] = rng.uniform(0.4, 0.9, 2).astype(np.float32)
            img = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
            pick = rng.integers(0, 3, (H, W))
            img[..., 3] = np.where(pick == 0, 0, np.where(pick == 1, 255, img[..., 3]))
            scene[f"image_{v}"] = img
            scene[f"normal_{v}"] = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        metas[f"scene_{s:03d}"] = scene
    return metas


class Cfg:
    def __init__(self, split, n_group, H, W, load_normal):
        self.data_root, self.split, self.img_size = "synthetic.h5", split, [H, W]
        self.n_scenes, self.n_group, self.load_normal = 3000000, n_group, load_normal


CASES = {
    # name: (split, n_group, H, W, load_normal, scene indices read in turn, seed)
    "train_g4": ("train", 4, 32, 32, True, (1, 0), 3),
    "test_g4": ("test", 4, 16, 16, True, (1,), 0),
    "train_g1": ("train", 1, 16, 16, True, (2,), 5),
    "train_g2": ("train", 2, 16, 16, True, (0,), 7),
    "nonsquare_train_g4": ("train", 4, 32, 48, True, (3,), 11),
    "test_no_normal": ("test", 4, 16, 32, False, (0,), 13),
}
SMALL = ("tar_c2w", "tar_w2c", "tar_ixt", "transform_mats", "bg_color", "near_far", "fovx", "fovy", "i2w", "i2w_down")


def seed_all(seed):
    random.seed(seed)
    torch.manual_seed(seed)


# ---- LaRa's own __getitem__, recorded ----

def _import_lara_gobjverse(lara, metas):
    """LaRa's dataLoader/gobjverse.py with a stub h5py whose File returns ``metas``."""
    h5 = types.ModuleType("h5py")
    h5.File = lambda path, mode="r": metas
    saved = {k: sys.modules.get(k) for k in ("h5py", "dataLoader", "dataLoader.utils", "dataLoader.gobjverse")}
    sys.modules["h5py"] = h5
    sys.modules["dataLoader"] = types.ModuleType("dataLoader")
    try:
        mods = {}
        for name in ("utils", "gobjverse"):
            spec = importlib.util.spec_from_file_location(f"dataLoader.{name}", os.path.join(lara, "dataLoader", f"{name}.py"))
            mods[name] = importlib.util.module_from_spec(spec)
            sys.modules[f"dataLoader.{name}"] = mods[name]
            spec.loader.exec_module(mods[name])
        return mods["gobjverse"], mods["utils"]
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def _with_i2w(fn, build_rays):
    """Run ``fn()`` and collect the ``i2ws`` local of every ``build_rays`` call it makes, as LaRa computed it."""
    seen = []

    def prof(frame, event, arg):
        if event == "return" and frame.f_code is build_rays.__code__:
            seen.append(np.array(frame.f_locals["i2ws"]))
    sys.setprofile(prof)
    try:
        out = fn()
    finally:
        sys.setprofile(None)
    return out, seen


def record_reference(lara, dev):
    """LaRa's ``gobjverse.__getitem__`` on the synthetic contents, run by this file's ``__main__``."""
    recs = {}
    for case, (split, g, H, W, nrm, indices, seed) in CASES.items():
        metas = synthetic_metas(seed, H, W)
        gob, utils = _import_lara_gobjverse(lara, metas)
        ds = gob.gobjverse(Cfg(split, g, H, W, nrm))
        seed_all(seed)
        for j, idx in enumerate(indices):
            s, i2ws = _with_i2w(lambda: ds[idx], utils.build_rays)
            assert len(i2ws) == 2
            r = {k: np.asarray(s[k]) for k in SMALL[:-2] + ("tar_rgb", "tar_msk", "tar_rays", "tar_rays_down")}
            if nrm:
                r["tar_nrm"] = s["tar_nrm"]
            r["i2w"], r["i2w_down"] = i2ws
            r["tar_view"] = np.array([int(v) for v in s["meta"]["tar_view"]])
            r["scene"] = np.array(s["meta"]["scene"])
            recs[f"{case}_{j}"] = r
    return recs


# ---- the torch CPU restatement of srf_batch_assemble ----

UNIT_U8 = torch.from_numpy(np.arange(256, dtype=np.float32) / np.float32(255))     # fp32(v / 255), NumPy's division


def _two_sum_err(a, b, s):
    bb = s - a
    return (a - (s - bb)) + (b - bb)


def _rays(i2w, origin, H, W, with_exact=False):
    """(rays [B,N,H,W,6] fp32, exact [B,N,H,W,3] bool): sum_j XYZ_j i2w[j][i] in fp64, j = 0, 1, 2, one rounding."""
    M = i2w.double()
    X = (torch.arange(W, dtype=torch.float64) + 0.5)[None, None, None, :]
    Y = (torch.arange(H, dtype=torch.float64) + 0.5)[None, None, :, None]
    dirs, exact = [], []
    for i in range(3):
        t0, t1, t2 = X * M[..., 0, i, None, None], Y * M[..., 1, i, None, None], M[..., 2, i, None, None].expand(-1, -1, H, W)
        s1 = t0 + t1
        s2 = s1 + t2
        dirs.append(s2.float())
        if with_exact:
            exact.append((_two_sum_err(t0, t1, s1) == 0) & (_two_sum_err(s1, t2, s2) == 0))
    o = origin[:, :, None, None, :].expand(-1, -1, H, W, -1)
    rays = torch.cat([o, torch.stack(dirs, -1)], -1)
    return rays, (torch.stack(exact, -1) if with_exact else None)


def normal_terms(nrm_u8, transform_mats):
    """(n [B,N,H,W,3] fp32 decoded normals, R [B,3,3], the fp64 terms t[..., i, j] = n_j R_ij, all exact)."""
    n = UNIT_U8[nrm_u8.long()] * 2 - 1
    R = transform_mats[:, 0, :3, :3]
    t = n.double()[..., None, :] * R.double()[:, None, None, None]
    return n, R, t


def assemble_reference(raw, with_exact=False):
    """What srf_batch_assemble writes, restated with torch on the CPU from a collated raw batch (host tensors)."""
    rgba = raw["tar_rgba"]
    B, N, H, W = rgba.shape[:4]
    c, a = UNIT_U8[rgba[..., :3].long()], UNIT_U8[rgba[..., 3:].long()]
    out = {"tar_rgb": c * a + raw["bg_color"][:, :, None, None, :] * (1 - a),
           "tar_msk": (rgba[..., 3] > 0).to(torch.uint8)}
    if raw.get("tar_nrm_u8") is not None:
        _, _, t = normal_terms(raw["tar_nrm_u8"], raw["transform_mats"])
        nrm = ((t[..., 0] + t[..., 1]) + t[..., 2]).float()
        out["tar_nrm"] = nrm.permute(0, 2, 1, 3, 4).reshape(B, H, N * W, 3)
    origin = raw["tar_c2w"][..., :3, 3]
    out["tar_rays"], ex = _rays(raw["i2w"], origin, H, W, with_exact)
    out["tar_rays_down"], exd = _rays(raw["i2w_down"], origin, H // 16, W // 16, with_exact)
    if with_exact:
        out["exact"], out["exact_down"] = ex, exd
    return out


def normal_bound(raw):
    """(float64 n R^T in tar_nrm's layout, sum_j |n_j R_ij| in the same layout)."""
    B, N, H, W = raw["tar_rgba"].shape[:4]
    _, _, t = normal_terms(raw["tar_nrm_u8"], raw["transform_mats"])
    lay = lambda v: v.permute(0, 2, 1, 3, 4).reshape(B, H, N * W, 3)     # noqa: E731
    return lay(t.sum(-1)), lay(t.abs().sum(-1))


GAMMA3 = 3 * U / (1 - 3 * U)    # any fp32 evaluation of a three-term dot product, in any order, FMA or not


def check_rays(got, want, exact, what):
    """Bit for bit where ``exact``; within one fp32 ulp of ``want`` elsewhere.  Returns the count of inexact sums."""
    got, want, exact = np.asarray(got), np.asarray(want), np.asarray(exact)
    assert got.shape == want.shape and got.dtype == want.dtype == np.float32, what
    assert np.array_equal(got[..., :3], want[..., :3]), f"{what}: origins"
    g, w = got[..., 3:], want[..., 3:]
    assert np.array_equal(g[exact], w[exact]), f"{what}: exact sums differ"
    ulp = np.spacing(np.maximum(np.abs(g), np.abs(w)).astype(np.float32))
    assert np.all(np.abs(g.astype(np.float64) - w) <= ulp), f"{what}: more than one ulp"
    return int((~exact).sum())


def check_against(out, raw, rec, b=0):
    """Scene ``b`` of ``out`` (assembled tensors) against LaRa's record ``rec`` under DESIGN §3.23's rules."""
    ref = assemble_reference(raw, with_exact=True)
    get = lambda k: out[k][b].cpu().numpy()       # noqa: E731
    assert np.array_equal(get("tar_rgb"), rec["tar_rgb"]) and get("tar_rgb").dtype == rec["tar_rgb"].dtype
    assert np.array_equal(get("tar_msk"), rec["tar_msk"]) and get("tar_msk").dtype == np.uint8
    n = check_rays(get("tar_rays"), rec["tar_rays"], ref["exact"][b].numpy(), "tar_rays")
    n += check_rays(get("tar_rays_down"), rec["tar_rays_down"], ref["exact_down"][b].numpy(), "tar_rays_down")
    if "tar_nrm" in rec:
        exact, mag = (v[b].numpy() for v in normal_bound(raw))
        # the assembly sums exact fp64 products and rounds once: within 2^-24 (1 + 2^-28) sum |t| < 2 * 2^-24 sum |t|;
        # LaRa's fp32 BLAS product is held to the general three-term bound
        for name, v, bound in (("assembled", get("tar_nrm"), 2 * U), ("LaRa's", rec["tar_nrm"], GAMMA3)):
            assert v.shape == exact.shape and v.dtype == np.float32
            assert np.all(np.abs(v - exact) <= bound * mag), f"{name} normals outside the bound"
    else:
        assert "tar_nrm" not in out
    return n


def collate(samples):
    return torch.utils.data.default_collate(samples)


def dataset_samples(case):
    """The GobjverseViews samples of a case, read in the record's order under the record's seeds."""
    from lara_b200.batch import GobjverseViews
    split, g, H, W, nrm, indices, seed = CASES[case]
    ds = GobjverseViews(Cfg(split, g, H, W, nrm), metas=synthetic_metas(seed, H, W))
    seed_all(seed)
    return [ds[i] for i in indices]


@pytest.mark.parametrize("case", list(CASES))
def test_dataset_equals_lara_record(case):
    samples = dataset_samples(case)
    metas = synthetic_metas(CASES[case][6], *CASES[case][2:4])
    for j, s in enumerate(samples):
        rec = reference_record("test_batch", f"{case}_{j}")
        assert [int(v) for v in s["meta"]["tar_view"]] == rec["tar_view"].tolist()
        assert s["meta"]["scene"] == rec["scene"]
        for k in SMALL:
            mine = np.asarray(s[k])
            assert mine.dtype == rec[k].dtype and mine.shape == rec[k].shape and np.array_equal(mine, rec[k]), k
        scene = metas[s["meta"]["scene"]]
        assert np.array_equal(s["tar_rgba"], np.stack([scene[f"image_{v}"] for v in s["meta"]["tar_view"]]))
        if CASES[case][4]:
            assert np.array_equal(s["tar_nrm_u8"], np.stack([scene[f"normal_{v}"] for v in s["meta"]["tar_view"]]))
        else:
            assert "tar_nrm_u8" not in s


@pytest.mark.parametrize("case", list(CASES))
def test_restatement_equals_lara_record(case):
    inexact = 0
    for j, s in enumerate(dataset_samples(case)):
        raw = collate([s])
        inexact += check_against(assemble_reference(raw), raw, reference_record("test_batch", f"{case}_{j}"))
    print(f"{case}: {inexact} ray components with an inexact fp64 sum (within one fp32 ulp)")


def test_record_covers_lara_branches():
    rec = reference_record("test_batch", "train_g4_0")
    assert set(np.unique(rec["bg_color"][4:])) <= {0.0, 0.5, 1.0} and np.all(rec["bg_color"][:4] == 1)
    assert rec["tar_rays_down"].shape == (8, 2, 2, 6) and rec["tar_nrm"].shape == (32, 8 * 32, 3)
    assert reference_record("test_batch", "train_g1_0")["tar_rgb"].shape[0] == 5
    assert reference_record("test_batch", "train_g2_0")["tar_rgb"].shape[0] == 4
    rec = reference_record("test_batch", "nonsquare_train_g4_0")
    assert rec["tar_rgb"].shape == (8, 32, 48, 3) and rec["tar_rays_down"].shape == (8, 2, 3, 6)
    assert rec["tar_ixt"][0, 0, 2] == 16.0 and rec["tar_ixt"][0, 1, 2] == 24.0     # cx from H, cy from W
    msk = rec["tar_msk"]
    assert msk.any() and not msk.all()


def test_dataset_rejects_what_is_not_uint8():
    from lara_b200.batch import GobjverseViews
    for key, dtype in (("image", np.float32), ("normal", np.int16)):
        metas = synthetic_metas(0, 16, 16)
        for s in metas.values():
            for v in range(12):
                s[f"{key}_{v}"] = s[f"{key}_{v}"].astype(dtype)
        with pytest.raises(TypeError, match=f"{key}_.* must be uint8"):
            GobjverseViews(Cfg("test", 4, 16, 16, True), metas=metas)[0]
    with pytest.raises(ValueError, match="expected"):
        GobjverseViews(Cfg("test", 4, 16, 32, False), metas=synthetic_metas(0, 16, 16))[0]


def test_assemble_batch_rejects_bad_inputs_before_any_launch():
    from lara_b200.batch import assemble_batch
    raw = collate(dataset_samples("test_g4"))
    with pytest.raises(TypeError, match="uint8"):
        assemble_batch({**raw, "tar_rgba": raw["tar_rgba"].float()})
    with pytest.raises(TypeError, match="uint8"):
        assemble_batch({**raw, "tar_nrm_u8": raw["tar_nrm_u8"].short()}, device="cuda:0")
    with pytest.raises(ValueError, match="tar_rgba"):
        assemble_batch({**raw, "tar_rgba": raw["tar_rgba"][..., :3]})
    with pytest.raises(RuntimeError, match="CUDA device"):
        assemble_batch(raw, device="cpu")


# ---- C entry: argument checks before any launch ----

def test_c_entry_rejects_bad_arguments_before_any_launch(lib):
    def call(B=1, N=2, H=16, W=16, rgba=256, normal=None, bg=512, i2w=768, i2w_down=1024, origin=1280, rot=None,
             rgb=4096, msk=8192, nrm=None, rays=12288, rays_down=16384):
        return lib.srf_batch_assemble(None, B, N, H, W, rgba, normal, bg, i2w, i2w_down, origin, rot, rgb, msk, nrm,
                                      rays, rays_down)
    for kw in ({"B": 0}, {"N": 0}, {"H": -1}, {"W": 0}, {"B": -3}):
        assert call(**kw) != 0 and b"bad sizes" in lib.srf_last_error(), kw
    for kw in ({"H": 15}, {"W": 15}, {"H": 8, "W": 64}):
        assert call(**kw) != 0 and b"at least 16" in lib.srf_last_error(), kw
    assert call(B=1 << 20, N=1 << 10, H=1 << 10, W=1 << 10) != 0 and b"too large" in lib.srf_last_error()
    for name in ("rgba", "bg", "i2w", "i2w_down", "origin", "rgb", "msk", "rays", "rays_down"):
        assert call(**{name: None}) != 0 and b"null" in lib.srf_last_error(), name
    for name in ("rgba", "bg", "i2w", "i2w_down", "origin", "rgb", "rays", "rays_down"):
        assert call(**{name: 258}) != 0 and b"aligned" in lib.srf_last_error(), name
    assert call(normal=2048, rot=None, nrm=20480) != 0 and b"nrm_rot" in lib.srf_last_error()
    assert call(normal=2048, rot=1536, nrm=None) != 0 and b"tar_nrm" in lib.srf_last_error()
    assert call(normal=2048, rot=1538, nrm=20480) != 0 and b"aligned" in lib.srf_last_error()


if __name__ == "__main__":
    # python tests/test_batch.py OUT_DIR LARA_CHECKOUT, then cp OUT_DIR/test_batch*.npz tests/golden/reference/
    spec = importlib.util.spec_from_file_location(
        "make_reference_records", os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                                               "make_reference_records.py"))
    writer = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(writer)
    os.makedirs(sys.argv[1], exist_ok=True)
    writer.save(sys.argv[1], "test_batch", record_reference(sys.argv[2], "cpu"))
