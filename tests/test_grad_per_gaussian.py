"""Every Gaussian's gradient, element by element, against a float64 replay of the forward's own blend decisions.

The replay (oracle/surfel_oracle.c: oracle_replay, oracle/oracle.py: replay / view_vjp / gaussian_grads) takes a
forward state -- records, tile lists, last and median contributors, contribution record -- recomputes the blend and
its backward in double, and carries for every output element a bound on what an fp32 evaluation of the same decisions
may differ by.  So a gradient is checked on its own scale, not against the largest gradient of the tensor: a wrong
factor in a path that only small gradients take (low-pass splats, the median terms, the background term, a tile's
last partial chunk) fails here.

CPU part: the replay is pinned against the C oracle's backward (another fp32 evaluation of the same decisions) and
against central finite differences of its own float64 forward.  GPU part: the kernels against the replay.
"""
import numpy as np
import pytest
import torch

from oracle import oracle as O

f64 = np.float64
CHANNELS = ["color", "depth", "alpha", "normal", "median_depth", "distortion", "median_weight"]


def _cam_dict(cam):
    return dict(viewmatrix=cam.viewmatrix.numpy().reshape(16), campos=cam.campos.numpy(), tanfovx=cam.tanfovx,
                tanfovy=cam.tanfovy, H=cam.image_height, W=cam.image_width)


def _oracle_state(run, sc_opacity):
    cb = (run.clamped.astype(np.int32) * np.array([1, 2, 4], np.int32)).sum(1)
    return dict(transMat=run.transMat, means2D=run.center, opacity=sc_opacity, normal=run.normal, rgb=run.rgb,
                ranges=run.ranges, point_list=run.point_list, n_contrib=run.n_contrib, contrib_masks=run.masks,
                clamp_bits=cb, visible=run.radii > 0)


def _upstream(H, W, seed, only=None):
    """Upstream gradients of magnitude ~1 per pixel; `only` keeps one output (colour, or one allmap channel group)."""
    g = np.random.default_rng(seed)
    gc = g.standard_normal((3, H, W)).astype(np.float32)
    ga = g.standard_normal((8, H, W)).astype(np.float32)
    if only is not None:
        keep = {"color": (), "depth": (0,), "alpha": (1,), "normal": (2, 3, 4), "median_depth": (5,),
                "distortion": (6,), "median_weight": (7,)}[only]
        if only != "color":
            gc[:] = 0
        for c in range(8):
            if c not in keep:
                ga[c] = 0
    return gc, ga


def _compare(got: dict, ref: dict, excl, ctx="", paths=None):
    """|got - ref| <= bound for every element of every output, Gaussians in `excl` aside.  Returns the worst ratio and
    where it is; `paths(i)` describes which blend paths Gaussian i's gradient comes from."""
    worst, where = 0.0, None
    for k, (v, e) in ref.items():
        if k not in got or got[k] is None:
            continue
        a = np.asarray(got[k], f64).reshape(v.shape)
        err = np.abs(a - v)
        keep = ~np.asarray(excl, bool).reshape((-1,) + (1,) * (v.ndim - 1))
        bad = (err > e) & keep
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.where(keep & (err > 0), err / e, 0.0)
        if ratio.size and ratio.max() > worst:
            worst = float(ratio.max())
            idx = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
            where = (k, tuple(int(i) for i in idx), float(a[idx]), float(v[idx]), float(e[idx]))
            if paths is not None:
                where += (paths(int(idx[0])),)
        assert not bad.any(), (f"{ctx} {k}: {int(bad.sum())} elements outside their bound; worst err/bound "
                               f"{ratio.max():.3g} at {where}")
    return worst, where


# ------------------------------------------------------------------------------------------------ CPU: the replay itself

def _oracle_case(P, seed, H, W, sh_degree, bg):
    from lara_b200 import scene as S
    sc = S.scene(P, seed, sh_degree)
    cam = S.cameras(2, H, W, seed)[0]
    run = O.run_scene(sc, cam, bg)
    return sc, cam, run


@pytest.mark.parametrize("sh_degree,bgv", [(1, 0.0), (3, 0.7), (0, 0.3)])
def test_replay_matches_the_oracle_backward(sh_degree, bgv):
    """The oracle's backward is another fp32 evaluation of its own forward's decisions: every gradient element, and
    every image pixel of the replay's forward, lies within the replay's bound of it.  Not within fp32 output rounding:
    the oracle sums in double, but it evaluates every pair in fp32 (backward.cu's own formulas), so it differs from
    the replay by the same per-pair rounding the bound is derived for."""
    sc, cam, run = _oracle_case(3000, sh_degree, 64, 80, sh_degree, torch.full((3,), bgv))
    st = _oracle_state(run, sc["opacities"].numpy().reshape(-1))
    gc, ga = _upstream(64, 80, sh_degree)
    r = O.replay(st, np.full(3, bgv, np.float32), gc, ga)
    img = np.concatenate([run.color, run.allmap, run.accum])
    assert (np.abs(img - r["img"]) <= r["img_e"]).all()
    og = run.backward(gc, ga)
    params = dict(means3D=sc["means3D"].numpy(), scales=sc["scales"].numpy(), rotations=sc["rotations"].numpy(),
                  shs=sc["shs"].numpy(), sh_degree=sh_degree)
    view = O.view_vjp(st, r["g"], r["g_e"], params, _cam_dict(cam))
    ref = O.gaussian_grads([view], params, st["opacity"])
    got = {"means3D": og["means3D"], "means2D": og["means2D"][:, :2], "sh": og["sh"], "opacities": og["opacities"],
           "scales": og["scales"], "rotations": og["rotations"], "transMat": og["transMat"]}
    assert r["pairs"] > 10_000
    worst, _ = _compare(got, ref, r["band"] != 0, "oracle")
    assert worst < 1.0


def _fd_scene(seed, sh_degree, raw):
    from lara_b200 import scene as S
    g = torch.Generator().manual_seed(seed)
    P = 40
    sc = S.scene(P, seed, sh_degree)
    sc["scales"] = sc["scales"] * 4.0
    sc["scales"][:8] *= 0.05                                  # sub-pixel splats: the low-pass branch
    sc["opacities"] = 0.2 + 0.7 * torch.rand((P, 1), generator=g)    # below the 0.99 clamp
    cam = S.cameras(2, 32, 32, seed, fov=0.9)[0]
    # one splat just beyond the near plane
    c2w = cam.c2w.double()
    sc["means3D"][8] = (c2w[:3, 3] + 0.25 * c2w[:3, 2]).float()
    sc["scales"][8] = 0.002
    return sc, cam


@pytest.mark.parametrize("sh_degree,raw", [(0, False), (1, True), (2, False), (3, True)])
def test_replay_gradients_are_finite_differences_of_its_forward(sh_degree, raw):
    """With the decisions held fixed, every checked replay gradient of a raw parameter agrees with the Richardson-
    extrapolated central difference of the replay's float64 forward (loss = <upstream, images>) to 1e-6 relative plus
    the double-rounding floor of the pixels the parameter touches; that floor is required to stay below a quarter of
    the gradient, so a sign error or a wrong factor fails on every element.  Non-raw rotations: the backward returns the
    gradient of the rotation polynomial at the unit quaternion, whose tangential part the normalising forward
    differentiates."""
    sc, cam = _fd_scene(10 + sh_degree, sh_degree, raw)
    bg = np.array([0.3, 0.1, 0.6], np.float32)
    run = O.run_scene(sc, cam, torch.from_numpy(bg))
    st = _oracle_state(run, sc["opacities"].numpy().reshape(-1))
    cd = _cam_dict(cam)
    P = sc["means3D"].shape[0]
    params = dict(means3D=sc["means3D"].numpy().astype(f64), shs=sc["shs"].numpy().astype(f64), sh_degree=sh_degree,
                  raw_activations=raw)
    if raw:
        params.update(scales=np.log(sc["scales"].numpy().astype(f64)), rotations=sc["rotations"].numpy().astype(f64) * 1.7,
                      opacities=np.log(sc["opacities"].numpy().astype(f64) / (1 - sc["opacities"].numpy())).reshape(-1))
    else:
        params.update(scales=sc["scales"].numpy().astype(f64), rotations=sc["rotations"].numpy().astype(f64),
                      opacities=sc["opacities"].numpy().reshape(-1).astype(f64))
    gc, ga = _upstream(32, 32, sh_degree)
    lp = np.zeros((max(run.num_rendered, 1), 256), np.uint8)
    rec, mult = O.preprocess64(params, cd, st["clamp_bits"])

    def state(rec):
        s = dict(st)
        s.update(rec)
        return s

    r = O.replay(state(rec), bg, gc, ga, lowpass=lp)
    assert r["lowpass_pairs"] > 20 and r["pairs"] > 500
    vis = st["visible"]
    assert vis[8] and r["npairs"][8] > 0                      # the splat at depth 0.25 is blended
    view = O.view_vjp(dict(st, transMat=rec["transMat"]), r["g"], r["g_e"], params, cd)
    ana = O.gaussian_grads([view], params, rec["opacity"])

    def weighted_images(p):
        """Per-pixel <upstream, images> of the replay's forward at parameters p, and the bound on its double rounding:
        the replay's fp32 bound img_e with the per-operation unit 2^-23 replaced by double's 2^-52."""
        rr = O.replay(state(O.preprocess64(p, cd, st["clamp_bits"], mult)[0]), bg, gc, ga, lowpass=lp, fix_lowpass=True)
        up = np.concatenate([gc, ga]).astype(f64)
        return up * rr["img"][:11], np.abs(up) * rr["img_e"][:11] * 2.0 ** -29

    def central(key, idx, h):
        """(L(p + h) - L(p - h)) / 2h summed per pixel: pixels the parameter does not touch cancel exactly, so the rounding
        floor is that of the touched pixels only."""
        pp = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in params.items()}
        pm = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in params.items()}
        pp[key][idx] += h
        pm[key][idx] -= h
        (wp, ep), (wm, em) = weighted_images(pp), weighted_images(pm)
        touched = wp != wm
        return float((wp - wm)[touched].sum()) / (2 * h), float((ep + em)[touched].sum()) / (2 * h)

    # Richardson extrapolation of two central differences (step h and h/2): truncation O(h^4), with h far below the
    # length over which each parameter changes the image (a pixel footprint for positions, the value itself for the
    # others), so that what remains is the rounding floor, derived per touched pixel above
    steps = {"means3D": 5e-5, "scales": 1e-3, "rotations": 1e-3, "opacities": 1e-3 if raw else 1e-4, "shs": 1e-2}
    names = {"shs": "sh"}
    checked, governed, worst = 0, 0, 0.0
    for key, h in steps.items():
        base = params[key]
        g_ana = ana[names.get(key, key)][0].reshape(base.shape)
        if key == "rotations" and not raw:
            qn = base / np.linalg.norm(base, axis=1, keepdims=True)
            g_ana = g_ana - qn * (g_ana * qn).sum(1, keepdims=True)
        for idx in np.ndindex(*base.shape):
            if not vis[idx[0]] or (idx[0] > 8 and idx[0] % 8):  # the small and near splats, an eighth of the rest
                continue
            if key == "shs" and (idx[1] >= (sh_degree + 1) ** 2 or idx[0] > 8):   # colour is linear in them
                continue
            hh = h * abs(base[idx]) if key == "scales" and not raw else h
            d1, n1 = central(key, idx, hh)
            d2, n2 = central(key, idx, hh / 2)
            fd, noise = (4 * d2 - d1) / 3, (4 * n2 + n1) / 3
            err = abs(fd - g_ana[idx])
            assert err <= 1e-6 * abs(g_ana[idx]) + noise, (key, idx, fd, g_ana[idx], noise)
            # the floor stays far below the gradient, so a sign error or a wrong factor fails on every element
            assert noise <= 0.25 * abs(g_ana[idx]), (key, idx, g_ana[idx], noise)
            worst = max(worst, err / abs(g_ana[idx]))
            governed += noise <= 1e-6 * abs(g_ana[idx])
            checked += 1
    print(f"{checked} gradient elements, worst |fd - g| / |g| {worst:.3g}; 1e-6 relative governs {governed}, the "
          f"rounding floor the rest")
    assert checked > 120


# ------------------------------------------------------------------------------------------------ GPU: kernel vs replay

def _run_kernel(sc, cam, bg, gc, ga, dev, raw=False, colors=None, transMat=None, params=None):
    from lara_b200 import rasterizer as R
    from lara_b200 import scene as S
    from lara_b200.debug import unpack_state
    st = S.settings_for(cam, torch.as_tensor(bg), sc["sh_degree"], dev, R.GaussianRasterizationSettings)
    p = params or sc
    t = lambda k: None if p.get(k) is None else torch.as_tensor(p[k]).float().to(dev).contiguous()
    shs = None if colors is not None else t("shs")
    cols = None if colors is None else torch.as_tensor(colors).float().to(dev)
    tm = None if transMat is None else torch.as_tensor(transMat).float().to(dev).contiguous()
    sca, rot = (None, None) if tm is not None else (t("scales"), t("rotations"))
    color, allmap, radii, state = R.forward_raw(t("means3D"), shs, cols, t("opacities"), sca, rot, tm, st,
                                                raw_activations=raw)
    g = R.backward_raw(state, radii, t("means3D"), shs, cols, sca, rot, tm, st, torch.as_tensor(gc).to(dev),
                       torch.as_tensor(ga).to(dev), raw_activations=raw)
    torch.cuda.synchronize()
    P = sc["means3D"].shape[0]
    u = {k: v.cpu().numpy() for k, v in unpack_state(state, P, cam.image_height, cam.image_width).items()}
    u["visible"] = radii.cpu().numpy() > 0
    out = {k: (None if v is None else v.cpu().numpy()) for k, v in g.items()}
    return u, out, np.concatenate([color.cpu().numpy(), allmap.cpu().numpy(), u["accum"]])


def _kernel_vs_replay(sc, cam, bg, gc, ga, dev, raw=False, colors=None, transMat=None, params=None, tiles=None):
    u, kg, img = _run_kernel(sc, cam, bg, gc, ga, dev, raw, colors, transMat, params)
    r = O.replay(u, bg, gc, ga, tiles=tiles)
    p = dict(params or {k: (v.numpy() if hasattr(v, "numpy") else v) for k, v in sc.items()})
    p["raw_activations"] = raw
    if colors is not None:
        p["shs"] = None
    view = O.view_vjp(u, r["g"], r["g_e"], p, _cam_dict(cam), precomp_T=transMat is not None,
                      precomp_colors=colors is not None)
    ref = O.gaussian_grads([view], p, u["opacity"], precomp_T=transMat is not None)
    got = {"means3D": kg["means3D"], "means2D": kg["means2D"][:, :2], "sh": kg.get("sh"),
           "opacities": kg["opacities"], "scales": None if transMat is not None else kg["scales"],
           "rotations": None if transMat is not None else kg["rotations"], "colors": kg.get("colors_precomp"),
           "transMat": kg.get("cov3Ds_precomp")}
    if tiles is None:
        assert (np.abs(img - r["img"]) <= r["img_e"]).all(), "forward images outside the replay's bound"
    band = r["band"] != 0
    nvis = max(int(u["visible"].sum()), 1)
    assert band.sum() < 1e-4 * nvis, f"{int(band.sum())} band Gaussians of {nvis} visible"
    npairs, nlow = r["npairs"], r["nlow"]
    paths = lambda i: f"{npairs[i]} pairs, {nlow[i]} low-pass, visible {bool(u['visible'][i])}"
    worst, where = _compare(got, ref, band, "kernel", paths)
    print(f"worst err/bound {worst:.3g} at {where}; band-excluded Gaussians {int(band.sum())}; pairs {r['pairs']}, "
          f"low-pass {r['lowpass_pairs']}")
    return r, u, worst


@pytest.fixture(scope="module")
def base_case():
    from lara_b200 import scene as S
    sc = S.scene(8000, 5)
    cam = S.cameras(3, 128, 144, 5)[0]
    return sc, cam


@pytest.mark.gpu
@pytest.mark.parametrize("only", CHANNELS + [None])
def test_kernel_gradients_one_output_at_a_time(cuda_device, base_case, only):
    sc, cam = base_case
    gc, ga = _upstream(128, 144, 1, only)
    r, u, worst = _kernel_vs_replay(sc, cam, np.array([0.2, 0.5, 0.9], np.float32), gc, ga, cuda_device)
    assert r["pairs"] > 100_000 and worst < 1.0


@pytest.mark.gpu
def test_kernel_gradients_sub_pixel_and_far_splats(cuda_device):
    from lara_b200 import scene as S
    sc = S.scene(20000, 6)
    sc["scales"] = sc["scales"] * 0.15
    sc["opacities"] = torch.full_like(sc["opacities"], 0.8)
    cam = S.cameras(3, 96, 112, 6, radius=3.5)[1]
    gc, ga = _upstream(96, 112, 2)
    r, _, _ = _kernel_vs_replay(sc, cam, np.array([0.1, 0.1, 0.1], np.float32), gc, ga, cuda_device)
    assert r["lowpass_pairs"] > 10_000 and r["lowpass_pairs"] > 0.5 * r["pairs"]


@pytest.mark.gpu
def test_kernel_gradients_at_the_footprint_switch(cuda_device):
    """Projected sigma ~0.707 px: rho3d ~ rho2d at every pixel, the pairs the exact re-evaluation band exists for."""
    from lara_b200 import scene as S
    sc = S.scene(30000, 7)
    cam = S.cameras(3, 128, 128, 7)[2]
    fx = 128 / (2 * cam.tanfovx)
    pv = sc["means3D"].double() @ cam.viewmatrix.double()[:3, :3] + cam.viewmatrix.double()[3, :3]
    sc["scales"] = (0.7071 * pv[:, 2:3] / fx).float().expand(-1, 2).contiguous()
    gc, ga = _upstream(128, 128, 3)
    r, _, _ = _kernel_vs_replay(sc, cam, np.zeros(3, np.float32), gc, ga, cuda_device)
    assert r["lowpass_pairs"] > 1000 and r["pairs"] - r["lowpass_pairs"] > 1000


@pytest.mark.gpu
def test_kernel_gradients_needles_and_saturation(cuda_device):
    from lara_b200 import scene as S
    sc = S.scene(20000, 3)
    sc["opacities"] = torch.full_like(sc["opacities"], 0.97)
    sc["scales"] = sc["scales"] * 2.5
    sc["scales"][::3, 1] *= 0.02                              # needles
    cam = S.cameras(3, 256, 200, 3)[1]
    gc, ga = _upstream(256, 200, 4)
    r, u, _ = _kernel_vs_replay(sc, cam, np.ones(3, np.float32), gc, ga, cuda_device)
    assert (u["accum"][0] < 1e-3).mean() > 0.5
    last = np.zeros((256, 208), np.int64)
    last[:, :200] = u["n_contrib"][0]
    blocks = last.reshape(64, 4, 26, 8).max((1, 3))
    lens = np.diff(u["ranges"], axis=1)[:, 0].reshape(16, 13)
    early = int((blocks.reshape(16, 4, 13, 2).transpose(0, 2, 1, 3).reshape(16, 13, 8) < lens[..., None]).sum())
    assert early > 100


@pytest.mark.gpu
def test_kernel_gradients_at_chunk_boundaries(cuda_device):
    """Tile lists of every length around the 16- and 32-entry chunks of the blend backward, and one of > 2048."""
    from lara_b200 import scene as S
    sc = S.scene(24000, 8)
    sc["scales"] = sc["scales"] * 0.2
    cl = slice(0, 2300)                                       # a cluster on one tile's centre
    cam = S.cameras(3, 320, 352, 8)[0]
    c2w = cam.c2w.double()
    fx = 352 / (2 * cam.tanfovx)
    ctr = c2w[:3, 3] + 1.905 * c2w[:3, 2] + (40.0 / fx * 1.905) * (c2w[:3, 0] + c2w[:3, 1])
    sc["means3D"][cl] = (ctr + 1e-3 * torch.randn(2300, 3, generator=torch.Generator().manual_seed(1)).double()).float()
    gc, ga = _upstream(320, 352, 5)
    r, u, _ = _kernel_vs_replay(sc, cam, np.array([0.5, 0.2, 0.1], np.float32), gc, ga, cuda_device)
    lens = set(np.diff(u["ranges"], axis=1)[:, 0].tolist())
    assert {1, 15, 16, 17, 31, 32, 33} <= lens and max(lens) > 2048, sorted(lens)


@pytest.mark.gpu
@pytest.mark.parametrize("sh_degree", [0, 1, 2, 3])
def test_kernel_gradients_ragged_and_sh_degrees(cuda_device, sh_degree):
    from lara_b200 import scene as S
    sc = S.scene(6000, 20 + sh_degree, sh_degree)
    cam = S.cameras(3, 77, 109, sh_degree)[1]
    gc, ga = _upstream(77, 109, 6)
    _kernel_vs_replay(sc, cam, np.array([0.9, 0.4, 0.2], np.float32), gc, ga, cuda_device)


@pytest.mark.gpu
def test_kernel_gradients_general_sh_rows(cuda_device):
    """M = 16 coefficient rows at degree 1: the general-M path, with rows beyond the degree zero."""
    from lara_b200 import scene as S
    sc = S.scene(5000, 30, 3)
    sc["sh_degree"] = 1
    cam = S.cameras(3, 96, 96, 2)[0]
    gc, ga = _upstream(96, 96, 7)
    _kernel_vs_replay(sc, cam, np.array([0.3, 0.3, 0.3], np.float32), gc, ga, cuda_device)


@pytest.mark.gpu
def test_kernel_gradients_colors_and_transmat_precomp(cuda_device):
    from lara_b200 import scene as S
    sc = S.scene(6000, 31, 2)
    cam = S.cameras(3, 96, 96, 3)[2]
    gc, ga = _upstream(96, 96, 8)
    cols = torch.rand((6000, 3), generator=torch.Generator().manual_seed(3))
    _kernel_vs_replay(sc, cam, np.array([0.3, 0.6, 0.3], np.float32), gc, ga, cuda_device, colors=cols.numpy())
    u, _, _ = _run_kernel(sc, cam, np.zeros(3, np.float32), gc, ga, cuda_device)
    tm = u["transMat"].copy()
    tm[~u["visible"]] = 0                                     # culled rows: anything
    _kernel_vs_replay(sc, cam, np.array([0.3, 0.6, 0.3], np.float32), gc, ga, cuda_device, transMat=tm)


@pytest.mark.gpu
def test_kernel_gradients_raw_activations(cuda_device):
    from lara_b200 import scene as S
    sc = S.scene(6000, 32, 1)
    cam = S.cameras(3, 96, 96, 4)[1]
    gc, ga = _upstream(96, 96, 9)
    o = sc["opacities"].numpy()
    p = dict(means3D=sc["means3D"].numpy(), shs=sc["shs"].numpy(), sh_degree=1, opacities=np.log(o / (1 - o)),
             scales=np.log(sc["scales"].numpy()), rotations=sc["rotations"].numpy() * 2.3)
    p["rotations"][:50] *= 1e-13                              # F.normalize's eps branch (norm < 1e-12)
    r, u, _ = _kernel_vs_replay(sc, cam, np.array([0.2, 0.2, 0.7], np.float32), gc, ga, cuda_device, raw=True, params=p)
    assert u["visible"][:50].sum() > 5


@pytest.mark.gpu
def test_kernel_gradients_of_three_views_with_accumulate(cuda_device):
    """forward_views_raw / backward_views_raw over V = 3 against the sum of the per-view replays, adding into a
    non-zero output buffer."""
    from lara_b200 import rasterizer as R
    from lara_b200 import scene as S
    from lara_b200.debug import unpack_state
    dev = cuda_device
    sc = S.scene(8000, 33, 1)
    cams = S.cameras(3, 80, 96, 9)
    bg = np.array([0.4, 0.1, 0.3], np.float32)
    settings = [S.settings_for(c, torch.from_numpy(bg), 1, dev, R.GaussianRasterizationSettings) for c in cams]
    camt = R.pack_cameras(settings, dev)
    t = {k: sc[k].to(dev).contiguous() for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    ups = [_upstream(80, 96, 40 + v) for v in range(3)]
    gc = torch.from_numpy(np.stack([u[0] for u in ups])).to(dev)
    ga = torch.from_numpy(np.stack([u[1] for u in ups])).to(dev)
    color, allmap, radii, state = R.forward_views_raw(t["means3D"], t["shs"], None, t["opacities"], t["scales"],
                                                      t["rotations"], None, camt, cams[0].tanfovx, cams[0].tanfovy,
                                                      80, 96, 1)
    P = 8000
    init = {k: torch.randn(s, generator=torch.Generator().manual_seed(i)).to(dev) * 1e-3 for i, (k, s) in
            enumerate([("means3D", (P, 3)), ("sh", (P, 4, 3)), ("opacities", (P, 1)), ("scales", (P, 2)),
                       ("rotations", (P, 4))])}
    out = {k: v.clone() for k, v in init.items()}
    R.backward_views_raw(state, radii, t["means3D"], t["shs"], None, t["scales"], t["rotations"], None, camt,
                         cams[0].tanfovx, cams[0].tanfovy, 80, 96, 1, gc, ga, out=out, accumulate=True)
    torch.cuda.synchronize()
    p = {k: (v.numpy() if hasattr(v, "numpy") else v) for k, v in sc.items()}
    views, band = [], np.zeros(P, bool)
    for v in range(3):
        u = {k: x.cpu().numpy() for k, x in unpack_state(state, P, 80, 96, view=v).items()}
        u["visible"] = radii[v].cpu().numpy() > 0
        r = O.replay(u, bg, ups[v][0], ups[v][1])
        views.append(O.view_vjp(u, r["g"], r["g_e"], p, _cam_dict(cams[v])))
        band |= r["band"] != 0
    ref = O.gaussian_grads(views, p, u["opacity"], out={k: v.cpu().numpy() for k, v in init.items()})
    got = {k: out[k].cpu().numpy() for k in ("means3D", "sh", "opacities", "scales", "rotations")}
    assert band.sum() < 1e-4 * P, f"{int(band.sum())} band Gaussians"
    worst, where = _compare(got, {k: ref[k] for k in got}, band, "views")
    print(f"worst err/bound {worst:.3g} at {where}; band-excluded Gaussians {int(band.sum())}")


@pytest.mark.gpu
def test_kernel_gradients_crop_at_the_bench_point(cuda_device):
    """131 072 Gaussians at 512 x 512 with upstream gradients on a crop of tiles only: the replay walks those tiles."""
    from lara_b200 import scene as S
    sc = S.scene(131072, 0)
    cam = S.cameras(8, 512, 512, 0)[0]
    gc, ga = _upstream(512, 512, 10)
    tiles = np.zeros((32, 32), bool)
    tiles[10:16, 12:20] = True
    pm = np.repeat(np.repeat(tiles, 16, 0), 16, 1)
    gc[:, ~pm] = 0
    ga[:, ~pm] = 0
    r, _, _ = _kernel_vs_replay(sc, cam, np.ones(3, np.float32), gc, ga, cuda_device, tiles=tiles.reshape(-1))
    assert r["pairs"] > 200_000
