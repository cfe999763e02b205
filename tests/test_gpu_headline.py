"""Parity at BASELINE.json's full sizes: the north-star point
(131 072 / 512^2), LaRa's own Gaussian count (524 288 / 512^2) and configs[3] (262 144 / 1024^2), all
against the recorded outputs of the UNMODIFIED reference build on an H100 (tests/golden/reference/, see
record_reference) -- radii and tile/sort indices bit for bit, colour and aux maps to fp32 rounding
(helpers.REF_FLOAT_TOL), gradients within helpers.REF_GRAD_TOL (or 10x the reference's own run-to-run atomic noise), over a
fixed sample of their elements -- plus a
fixed-seed 25-configuration slice of tools/parity_sweep.py (ragged sizes, SH degrees 0-3, needle splats,
saturated scenes, cameras inside the cloud)."""
import numpy as np
import pytest
import torch

from helpers import (REF_GRAD_TOL, allmap_records, compare_records, count_record, fingerprint, reference_record, rel_err, run_candidate,
                     sampled_rel_err, tile_pixel_mask, to_dev, tolerance_record)

pytestmark = pytest.mark.gpu

HEADLINE = [  # P, size, seed
    (131072, 512, 0),
    (524288, 512, 1),
    (262144, 1024, 2),
]
GRAD_KEYS = (("g_means3D", "means3D"), ("g_sh", "shs"), ("g_opacities", "opacities"), ("g_scales", "scales"),
             ("g_rotations", "rotations"))


# record sizes of a sweep configuration (helpers.tolerance_record): 25 of them share one record file
SWEEP_IMAGE = {"n": 128, "blocks": 128}
SWEEP_GRAD = {"n": 256, "blocks": 256}
SWEEP_COUNTS = 512


def _state(r, H, W, image_kw=None, counts=1024):
    """Integer state as fingerprints, images (aux maps per channel) and per-pixel counts as records."""
    image_kw = image_kw or {}
    m = tile_pixel_mask(r["ranges"], H, W)
    rec = {k: fingerprint(r[k]) for k in ("radii", "point_list", "ranges")}
    rec["num_rendered"] = int(r["num_rendered"])
    rec.update({k: tolerance_record(r[k], **image_kw) for k in ("color", "accum")})
    rec.update(allmap_records(r["allmap"], **image_kw))
    rec["n_contrib"] = count_record(r["n_contrib"][0], counts)
    rec["median_contributor"] = count_record(r["n_contrib"][1][m], counts)
    return rec


def _reference_record(ref, sc, cam, bg, deg, dev, gc, ga, twice=False, sweep=False):
    """The reference's state fingerprints and gradient records (with its run-to-run noise when `twice`)."""
    from lara_b200 import scene as S
    from oracle import ref as REF
    scd = to_dev(sc, dev)
    st = S.settings_for(cam, bg, deg, dev, ref.GaussianRasterizationSettings)
    r = REF.forward_raw(ref, scd, st)
    r = {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in r.items()}

    def grads():
        leaves = {k: scd[k].clone().requires_grad_(True) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
        rast = ref.GaussianRasterizer(raster_settings=st)
        c_, rd_, am_ = rast(means3D=leaves["means3D"], means2D=torch.zeros_like(leaves["means3D"]), shs=leaves["shs"],
                            opacities=leaves["opacities"], scales=leaves["scales"], rotations=leaves["rotations"])
        torch.autograd.backward((c_, am_), (gc.to(dev), ga.to(dev)))
        return {k: v.grad.cpu().numpy() for k, v in leaves.items()}
    g1 = grads()
    g2 = grads() if twice else g1
    rec = _state(r, cam.image_height, cam.image_width, *((SWEEP_IMAGE, SWEEP_COUNTS) if sweep else ()))
    for _, b_ in GRAD_KEYS:
        rec[b_] = tolerance_record(g1[b_], **(SWEEP_GRAD if sweep else {}))
        rec["noise_" + b_] = rel_err(g2[b_], g1[b_])
    return rec


def _compare(mine, rec, H, W, sweep=False):
    errs = compare_records(_state(mine, H, W, *((SWEEP_IMAGE, SWEEP_COUNTS) if sweep else ())), rec)
    worst = 0.0
    for a_, b_ in GRAD_KEYS:
        e = sampled_rel_err(mine[a_], rec, b_)
        noise = float(rec["noise_" + b_])
        worst = max(worst, e)
        if not (np.isfinite(mine[a_]).all() and e < max(REF_GRAD_TOL, 10 * noise)):
            errs.append(f"grad_{b_}({e:.1e}, ref noise {noise:.1e})")
    return errs, worst


def record_reference(ref, dev):
    """The reference's side of the comparisons below (tests/golden/make_reference_records.py)."""
    from lara_b200 import scene as S
    out = {}
    for P, size, seed in HEADLINE:
        sc, cam, bg = _headline_inputs(P, size, seed)
        gc, ga = S.upstream_grads(size, size, seed)
        out[f"headline/{P}-{size}-{seed}"] = _reference_record(ref, sc, cam, bg, 1, dev, gc, ga, twice=True)
    rng = np.random.default_rng(SWEEP_SEED)
    for it in range(25):
        tag, sc, cam = _sweep_config(rng)
        gc, ga = S.upstream_grads(tag["H"], tag["W"], tag["seed"])
        out[f"sweep/{it}"] = _reference_record(ref, sc, cam, torch.full((3,), tag["bg"]), tag["deg"], dev, gc, ga,
                                               sweep=True)
    return out


def _headline_inputs(P, size, seed):
    from lara_b200 import scene as S
    return S.scene(P, seed, sh_degree=1), S.cameras(3, size, size, seed)[seed % 3], torch.ones(3)


@pytest.mark.parametrize("P,size,seed", HEADLINE)
def test_headline_sizes_vs_reference(cuda_device, P, size, seed):
    from lara_b200 import scene as S
    sc, cam, bg = _headline_inputs(P, size, seed)
    gc, ga = S.upstream_grads(size, size, seed)
    mine = run_candidate(sc, cam, bg, cuda_device, grads=(gc, ga))
    errs, worst = _compare(mine, reference_record("test_gpu_headline", f"headline/{P}-{size}-{seed}"), size, size)
    assert not errs, (errs, worst)
    assert mine["num_rendered"] > P          # the configuration really has LaRa-like overdraw


def _sweep_config(rng):
    from lara_b200 import scene as S
    P = int(rng.choice([500, 3000, 20000, 60000, 150000, 300000]))
    H = int(rng.choice([64, 100, 200, 256, 333, 512, 768])); W = int(rng.choice([64, 120, 200, 256, 400, 512, 700]))
    deg = int(rng.integers(0, 4)); bgv = float(rng.choice([0.0, 0.5, 1.0])); seed = int(rng.integers(0, 10000))
    sc = S.scene(P, seed, sh_degree=deg)
    sc["scales"] = sc["scales"] * float(rng.choice([0.3, 1.0, 2.5, 6.0]))
    if rng.random() < 0.3:
        sc["scales"][:, 1] *= 0.05                      # needle-like splats (edge-on conics)
    if rng.random() < 0.3:
        sc["opacities"] = torch.rand(sc["opacities"].shape, generator=torch.Generator().manual_seed(seed))   # saturation
    fov = float(rng.choice([0.4, 0.75, 1.3])); radius = float(rng.choice([0.9, 1.905, 4.0]))   # 0.9: camera inside the cloud
    cam = S.cameras(3, H, W, seed, fov=fov, radius=radius)[seed % 3]
    return dict(P=P, H=H, W=W, deg=deg, bg=bgv, seed=seed, fov=fov, radius=radius), sc, cam


SWEEP_SEED = 20260924


def test_parity_sweep_slice_25_configurations(cuda_device):
    from lara_b200 import scene as S
    rng = np.random.default_rng(SWEEP_SEED)
    failures, worst = [], 0.0
    for it in range(25):
        tag, sc, cam = _sweep_config(rng)
        bg = torch.full((3,), tag["bg"])
        gc, ga = S.upstream_grads(tag["H"], tag["W"], tag["seed"])
        mine = run_candidate(sc, cam, bg, cuda_device, grads=(gc, ga))
        errs, w = _compare(mine, reference_record("test_gpu_headline", f"sweep/{it}"), tag["H"], tag["W"], sweep=True)
        worst = max(worst, w)
        if errs:
            failures.append((tag, errs))
    assert not failures, (failures, worst)
