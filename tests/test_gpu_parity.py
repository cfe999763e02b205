"""GPU parity of the CUDA path, through the C ABI:
  * against the recorded outputs of the UNMODIFIED reference build on an H100 (tests/golden/reference/,
    see record_reference): radii, tiles and tile/sort indices bit-exact, floats to fp32 rounding
    (helpers.REF_FLOAT_TOL: the reference rounds differently per architecture), gradients within 1e-4
    (the reference's own run-to-run atomic noise is ~1e-6),
  * against the CPU oracle and the committed golden fixtures (bit-exact: the reference's sm_100 outputs)."""
import numpy as np
import pytest
import torch

from helpers import (allmap_records, compare_records, count_record, fingerprint, golden_files, load_golden, reference_record, rel_err, run_candidate,
                     sampled_rel_err, scene_from_golden, tile_pixel_mask, to_dev, tolerance_record)

pytestmark = pytest.mark.gpu

# see tests/test_oracle_golden.py: the distortion channel is ill-conditioned in fp32 (CPU vs GPU only)
ALLMAP_TOL = [1e-4, 1e-4, 1e-4, 1e-4, 1e-4, 1e-4, 5e-3, 1e-4]

CASES = [  # P, H, W, seed, sh_degree, bg
    (4096, 128, 128, 0, 1, 1.0),
    (6000, 300, 500, 1, 3, 0.5),     # not multiples of 16, degree-3 SH
    (20000, 256, 256, 2, 0, 0.0),
    (32768, 512, 512, 3, 1, 1.0),    # BASELINE configs[1]
    (50000, 200, 200, 4, 2, 0.5),    # many instances per tile (> 2048: big-tile sort path)
]


def _case_id(c):
    return "-".join(str(x) for x in c)


def _case_inputs(P, H, W, seed, deg, bgv):
    from lara_b200 import scene as S
    return S.scene(P, seed, sh_degree=deg), S.cameras(3, H, W, seed)[seed % 3], torch.full((3,), bgv)


def _forward_state(r, H, W):
    """Record of the forward: integer state as fingerprints, floats and per-pixel counts as samples."""
    vis = r["radii"] > 0
    mask = tile_pixel_mask(r["ranges"], H, W)   # reference leaves empty tiles' median plane uninitialised
    rec = {k: fingerprint(r[k]) for k in ("radii", "tiles_touched", "point_list", "ranges")}
    rec["num_rendered"] = int(r["num_rendered"])
    rec.update({k: tolerance_record(r[k][vis]) for k in ("depths", "transMat", "means2D", "rgb")})
    rec.update({k: tolerance_record(r[k]) for k in ("accum", "color")})
    rec.update(allmap_records(r["allmap"]))
    rec["n_contrib"] = count_record(r["n_contrib"][0])
    rec["median_contributor"] = count_record(r["n_contrib"][1][mask])
    return rec


def record_reference(ref, dev):
    """The reference's side of the comparisons below (tests/golden/make_reference_records.py)."""
    from lara_b200 import scene as S
    from oracle import ref as REF
    out = {}
    for c in CASES:
        P, H, W, seed, deg, bgv = c
        sc, cam, bg = _case_inputs(*c)
        scd = to_dev(sc, dev)
        st = S.settings_for(cam, bg, deg, dev, ref.GaussianRasterizationSettings)
        r = REF.forward_raw(ref, scd, st)
        r = {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in r.items()}
        out["state/" + _case_id(c)] = _forward_state(r, H, W)
    for c in CASES[:4]:
        P, H, W, seed, deg, bgv = c
        sc, cam, bg = _case_inputs(*c)
        scd = to_dev(sc, dev)
        gc, ga = [t.to(dev) for t in S.upstream_grads(H, W, seed)]
        st = S.settings_for(cam, bg, deg, dev, ref.GaussianRasterizationSettings)
        gr, gr2 = _autograd_grads(ref, scd, st, gc, ga), _autograd_grads(ref, scd, st, gc, ga)
        rec = {k: tolerance_record(gr[k]) for k in gr}
        rec.update({"noise_" + k: rel_err(gr2[k], gr[k]) for k in gr})
        out["grads/" + _case_id(c)] = rec
    return out


def _autograd_grads(mod, scd, st, gc, ga):
    leaves = {k: scd[k].clone().requires_grad_(True) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    m2d = torch.zeros_like(leaves["means3D"], requires_grad=True)
    rast = mod.GaussianRasterizer(raster_settings=st)
    c, rd, am = rast(means3D=leaves["means3D"], means2D=m2d, shs=leaves["shs"], opacities=leaves["opacities"],
                     scales=leaves["scales"], rotations=leaves["rotations"])
    torch.autograd.backward((c, am), (gc, ga))
    g = {k: v.grad.detach().cpu().numpy() for k, v in leaves.items()}
    g["means2D"] = m2d.grad.detach().cpu().numpy()
    return g


@pytest.mark.parametrize("P,H,W,seed,deg,bgv", CASES)
def test_forward_state_bit_exact_vs_reference(cuda_device, P, H, W, seed, deg, bgv):
    sc, cam, bg = _case_inputs(P, H, W, seed, deg, bgv)
    mine = _forward_state(run_candidate(sc, cam, bg, cuda_device), H, W)
    rec = reference_record("test_gpu_parity", "state/" + _case_id((P, H, W, seed, deg, bgv)))
    # point_list is the sort order incl. ties, rgb pins the SH evaluation, allmap all 8 aux maps
    assert not compare_records(mine, rec)


@pytest.mark.parametrize("P,H,W,seed,deg,bgv", CASES[:4])
def test_gradients_vs_reference(cuda_device, P, H, W, seed, deg, bgv):
    import diff_surfel_rasterization as DSR
    from lara_b200 import scene as S
    sc, cam, bg = _case_inputs(P, H, W, seed, deg, bgv)
    scd = to_dev(sc, cuda_device)
    gc, ga = [t.to(cuda_device) for t in S.upstream_grads(H, W, seed)]
    st_m = S.settings_for(cam, bg, deg, cuda_device, DSR.GaussianRasterizationSettings)
    with torch.autograd.set_detect_anomaly(True):      # LaRa trains with anomaly mode on
        gm = _autograd_grads(DSR, scd, st_m, gc, ga)
    rec = reference_record("test_gpu_parity", "grads/" + _case_id((P, H, W, seed, deg, bgv)))
    for k in gm:
        assert np.isfinite(gm[k]).all(), k
        noise = float(rec["noise_" + k])
        err = sampled_rel_err(gm[k], rec, k)
        assert err < max(1e-4, 10 * noise), (k, err, noise)
    assert gm["opacities"].shape == (P, 1) and gm["means2D"].shape == (P, 3)
    assert float(np.abs(gm["means2D"][:, 2]).max()) == 0.0


@pytest.mark.parametrize("P,H,W,seed,deg,bgv", [(2048, 64, 64, 0, 1, 1.0), (3000, 50, 72, 1, 3, 0.5), (1500, 96, 96, 5, 2, 0.0)])
def test_candidate_vs_cpu_oracle(cuda_device, P, H, W, seed, deg, bgv):
    from lara_b200 import scene as S
    from oracle import oracle as O
    sc = S.scene(P, seed, sh_degree=deg)
    cam = S.cameras(3, H, W, seed)[seed % 3]
    bg = torch.full((3,), bgv)
    gc, ga = S.upstream_grads(H, W, seed)
    mine = run_candidate(sc, cam, bg, cuda_device, grads=(gc, ga))
    run = O.run_scene(sc, cam, bg)
    og = run.backward(gc, ga)
    assert int((mine["radii"] != run.radii).sum()) <= max(1, P // 500)
    assert rel_err(mine["color"], run.color) < 1e-4
    for c in range(8):
        assert rel_err(mine["allmap"][c], run.allmap[c]) < ALLMAP_TOL[c], c
    for a, b in (("g_means3D", "means3D"), ("g_sh", "sh"), ("g_opacities", "opacities"), ("g_scales", "scales"),
                 ("g_rotations", "rotations"), ("g_means2D", "means2D")):
        assert rel_err(mine[a], og[b]) < 1e-4, a
    run.close()


@pytest.mark.parametrize("path", golden_files(), ids=lambda p: p.split("/")[-1][:-4])
def test_candidate_vs_golden_fixtures(cuda_device, path):
    """Same checks as against the live reference, but from the committed reference outputs."""
    z = load_golden(path)
    sc, cam, bg = scene_from_golden(z)
    H, W = int(z["H"]), int(z["W"])
    mine = run_candidate(sc, cam, bg, cuda_device, grads=(torch.from_numpy(z["grad_color"]), torch.from_numpy(z["grad_allmap"])))
    assert np.array_equal(mine["radii"], z["radii"])
    assert np.array_equal(mine["tiles_touched"], z["tiles_touched"])
    assert mine["num_rendered"] == int(z["num_rendered"])
    assert np.array_equal(mine["point_list"], z["point_list"])
    assert np.array_equal(mine["ranges"], z["ranges"])
    assert np.array_equal(mine["n_contrib"][0], z["n_contrib"][0])
    assert np.array_equal(mine["allmap"].view(np.int32), z["allmap"].view(np.int32))
    assert np.array_equal(mine["color"].view(np.int32), z["color"].view(np.int32))
    for a, b in (("g_means3D", "g_means3D"), ("g_sh", "g_shs"), ("g_opacities", "g_opacities"), ("g_scales", "g_scales"),
                 ("g_rotations", "g_rotations"), ("g_means2D", "g_means2D")):
        assert rel_err(mine[a], z[b]) < 1e-4, a
