"""Shared test helpers (not a test module)."""
from __future__ import annotations

import glob
import hashlib
import os

import numpy as np
import torch

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden_files():
    return sorted(glob.glob(os.path.join(GOLDEN_DIR, "*.npz")))


# ---- records of the reference rasterizer's outputs (tests/golden/reference/<module>.npz) ----
# Written by tests/golden/make_reference_records.py from each test module's record_reference().  Arrays the
# tests compare bit for bit are kept as fingerprints.  An array compared with a tolerance is kept as its absolute
# maximum (the denominator of rel_err), a fixed, seeded sample of its elements, and the maximum and minimum of each
# of BLOCKS contiguous blocks of it: a block's extremes move by at most max|a - b| over the block, so they obey the
# same tolerance as the elements, and together they cover every element.
REFERENCE_DIR = os.path.join(GOLDEN_DIR, "reference")
SAMPLE = 1024
BLOCKS = 512


_FLOAT_BITS = {np.dtype(np.float16): np.int16, np.dtype(np.float32): np.int32, np.dtype(np.float64): np.int64}


def fingerprint(a) -> str:
    """Digest of an array's values and shape: integers and booleans compared as int64, floats by their bits."""
    a = np.ascontiguousarray(a)
    if a.dtype.kind == "f":
        if a.dtype not in _FLOAT_BITS:
            raise TypeError(f"fingerprint: no bit-exact view for {a.dtype}")
        a = a.view(_FLOAT_BITS[a.dtype])
    elif a.dtype.kind not in "biu":
        raise TypeError(f"fingerprint: not a numeric array ({a.dtype})")
    a = np.ascontiguousarray(a.astype(np.int64))
    return hashlib.sha256(repr(a.shape).encode() + a.tobytes()).hexdigest()[:40]


def sample(a, n=SAMPLE):
    """Fixed, seeded sample of n elements of the flattened array (all of them if it is smaller)."""
    flat = np.asarray(a, dtype=np.float64).reshape(-1)
    if flat.size <= n:
        return flat
    return flat[np.sort(np.random.default_rng(0).choice(flat.size, n, replace=False))]


def tolerance_record(a, n=SAMPLE, blocks=BLOCKS):
    a = np.asarray(a, dtype=np.float64)
    flat = a.reshape(-1)
    rec = {"sample": sample(a, n).astype(np.float32), "absmax": float(np.abs(flat).max()) if flat.size else 0.0,
           "shape": np.array(a.shape)}
    if flat.size > n:          # else the sample is the whole array
        starts = np.linspace(0, flat.size, min(blocks, flat.size) + 1).astype(np.int64)[:-1]
        rec["bmax"] = np.maximum.reduceat(flat, starts).astype(np.float32)
        rec["bmin"] = np.minimum.reduceat(flat, starts).astype(np.float32)
    return rec


def record_error(v, rec, key) -> float:
    """Largest difference between the record `v` and the recorded reference `key` (sample and block extremes),
    relative to the reference's absolute maximum (at least REF_SCALE_FLOOR of the key)."""
    m = max(float(rec[key + ".absmax"]), REF_SCALE_FLOOR.get(key.rsplit("/", 1)[-1], 0.0))
    d = 0.0
    for f in ("sample", "bmax", "bmin"):
        if key + "." + f in rec:
            x = np.abs(np.asarray(v[f], dtype=np.float64) - rec[key + "." + f])
            d = max(d, float(x.max()) if x.size else 0.0)
    return d / (m if m > 0 else 1.0)


def sampled_rel_err(a, rec, key) -> float:
    """rel_err of `a` against the recorded reference array `key`, over its recorded sample and block extremes."""
    assert tuple(np.asarray(a).shape) == tuple(rec[key + ".shape"]), key
    blocks = rec[key + ".bmax"].size if key + ".bmax" in rec else BLOCKS
    return record_error(tolerance_record(a, rec[key + ".sample"].size, blocks), rec, key)


def allmap_records(allmap, **kw):
    """Tolerance records of the 8 aux maps, one per channel: each is compared relative to its own maximum."""
    return {f"allmap{c}": tolerance_record(np.asarray(allmap)[c], **kw) for c in range(8)}


def count_record(a, n=1024):
    """Integer map compared element by element over a fixed sample."""
    a = np.asarray(a)
    return {"sample": sample(a, n).astype(np.int32), "shape": np.array(a.shape)}


# The reference's fp32 arithmetic depends on the architecture it is compiled for: nvcc contracts its expressions
# into FMAs differently for sm_90 and sm_100.  This package keeps the operation order of the reference's sm_100
# build (bit for bit against tests/golden/*.npz, test_candidate_vs_golden_fixtures).  Against the reference's
# sm_90 build (the records) float outputs agree to REF_FLOAT_TOL of the array's maximum, and per-pixel counts
# except where the transmittance lands within rounding of its stopping threshold.  The distortion map (aux channel 6)
# sums terms w * (m^2 A + D2 - 2 m D1) with weights and mapped depths below 1 that cancel to ~1e-6
# (tests/test_oracle_golden.py): it gets 5e-3 of its maximum, and a map whose maximum is far below its terms is
# cancellation residue, so its scale is floored at REF_SCALE_FLOOR.  Gradients: where the two builds' rounding takes
# a different accept / stop decision for a pair near a threshold, that pair's splat moves by up to ~5e-4 of the
# gradient's maximum (measured over the sweep of tests/test_gpu_headline.py): REF_GRAD_TOL.
REF_FLOAT_TOL = 1e-5
REF_TOL = {"allmap6": 5e-3}
REF_SCALE_FLOOR = {"allmap6": 1e-4}
REF_GRAD_TOL = 1e-3


def compare_records(mine: dict, rec: dict, tol=None) -> list:
    """Names of the fields of `mine` (built like the record) that do not match the recorded reference."""
    tol = tol or {}
    bad = []
    for k, v in mine.items():
        if isinstance(v, dict):
            if tuple(v["shape"]) != tuple(rec[k + ".shape"]):
                bad.append(k)
            elif "absmax" in v:
                e = record_error(v, rec, k)
                if not e <= tol.get(k, REF_TOL.get(k, REF_FLOAT_TOL)):
                    bad.append(f"{k}({e:.1e})")
            elif int((v["sample"] != rec[k + ".sample"]).sum()) > max(2, v["sample"].size // 200):
                bad.append(k)
        elif v != (int(rec[k]) if isinstance(v, int) else rec[k]):
            bad.append(k)
    return bad


def flatten_record(rec: dict) -> dict:
    out = {}
    for k, v in rec.items():
        if isinstance(v, dict):
            out.update({f"{k}.{kk}": vv for kk, vv in v.items()})
        else:
            out[k] = v
    return out


def reference_record(module: str, case: str) -> dict:
    """The recorded reference outputs of one case of a test module (<module>.npz, <module>.1.npz, ...)."""
    pre = case + "/"
    rec = {}
    for path in [os.path.join(REFERENCE_DIR, module + ".npz")] + glob.glob(os.path.join(REFERENCE_DIR, module + ".*.npz")):
        z = np.load(path)
        rec.update({k[len(pre):]: z[k] for k in z.files if k.startswith(pre)})
    assert rec, f"no reference record for {module} {case}"
    return {k: (str(v) if v.dtype.kind == "U" else v) for k, v in rec.items()}


SEEDED_INPUTS = ("means3D", "scales", "rotations", "opacities", "shs", "grad_color", "grad_allmap")


def load_golden(path) -> dict:
    """A golden fixture.  A file that names its `case` leaves out the inputs make_golden.case_inputs() regenerates
    bit for bit from seeds (the scene and the upstream gradients), which keeps it small."""
    z = dict(np.load(path))
    if "case" in z:
        import sys
        sys.path.insert(0, GOLDEN_DIR)
        from make_golden import case_inputs, upstream_grads_for
        sc, cam, _ = case_inputs(str(z["case"]))
        gc, ga = upstream_grads_for(cam)
        z.update({k: sc[k].numpy() for k in SEEDED_INPUTS[:5]})
        z.update(grad_color=gc.numpy(), grad_allmap=ga.numpy())
    return z


def rel_err(a, b) -> float:
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    if a.size == 0:
        return 0.0
    m = np.abs(b).max()
    return float(np.abs(a - b).max() / (m if m > 0 else 1.0))


def to_dev(sc, dev):
    return {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in sc.items()}


def tile_pixel_mask(ranges, H, W):
    """[H,W] bool: pixel lies in a tile whose range is non-empty (the reference leaves the median
    contributor plane uninitialised for empty tiles)."""
    gx = (W + 15) // 16
    nonempty = (ranges[:, 1] > ranges[:, 0])
    ty = np.arange(H) // 16
    tx = np.arange(W) // 16
    return nonempty[(ty[:, None] * gx + tx[None, :])]


def run_candidate(sc, cam, bg, dev, grads=None, debug=False):
    """Candidate forward (+ backward if grads=(gc,ga)) through the raw API; returns a dict of
    CPU numpy arrays including the internal state."""
    from lara_b200 import rasterizer as R
    from lara_b200 import scene as S
    from lara_b200.debug import unpack_state
    scd = to_dev(sc, dev)
    st = S.settings_for(cam, bg, sc["sh_degree"], dev, R.GaussianRasterizationSettings, debug=debug)
    H, W = cam.image_height, cam.image_width
    P = sc["means3D"].shape[0]
    color, allmap, radii, state = R.forward_raw(scd["means3D"], scd.get("shs"), scd.get("colors_precomp"),
                                                scd["opacities"], scd["scales"], scd["rotations"], None, st)
    torch.cuda.synchronize()
    u = unpack_state(state, P, H, W)
    out = {"color": color, "allmap": allmap, "radii": radii, "num_rendered": state.num_rendered}
    out.update({k: u[k] for k in ("ranges", "point_list", "n_contrib", "accum")})
    if P > 0:
        out.update({k: u[k] for k in ("tiles_touched", "depths", "transMat", "means2D", "rgb", "normal")})
    if grads is not None:
        gc, ga = grads
        g = R.backward_raw(state, radii, scd["means3D"], scd.get("shs"), scd.get("colors_precomp"), scd["scales"],
                           scd["rotations"], None, st, gc.to(dev), ga.to(dev))
        torch.cuda.synchronize()
        out.update({"g_" + k: v for k, v in g.items() if v is not None})
    return {k: (v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in out.items()}


def scene_from_golden(z):
    sc = {"means3D": torch.from_numpy(z["means3D"]), "scales": torch.from_numpy(z["scales"]),
          "rotations": torch.from_numpy(z["rotations"]), "opacities": torch.from_numpy(z["opacities"]),
          "shs": torch.from_numpy(z["shs"]), "sh_degree": int(z["sh_degree"])}
    from lara_b200.scene import Camera
    cam = Camera(int(z["H"]), int(z["W"]), float(z["tanfovx"]), float(z["tanfovy"]),
                 torch.from_numpy(z["viewmatrix"]), torch.from_numpy(z["projmatrix"]), torch.from_numpy(z["campos"]),
                 torch.eye(4))
    return sc, cam, torch.from_numpy(z["bg"])
