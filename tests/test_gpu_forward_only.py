"""Forward-only rendering on the GPU: the forward-only blend (no contribution record, no image state) gives the training
forward's outputs bit for bit -- through the raw entries, the drop-in wrappers, render_scene_views and the Renderer --
repairs an overflowed capacity the same way, needs at least the record's bytes less memory, and leaves a training
forward's pending backward untouched."""
import math
import warnings
from typing import NamedTuple

import pytest
import torch

from helpers import to_dev

pytestmark = pytest.mark.gpu

KEYS = ("means3D", "shs", "opacities", "scales", "rotations")


def _scene(P, deg, seed, kind="lara"):
    from lara_b200 import scene as S
    sc = S.scene(P, seed, sh_degree=deg)
    if kind == "saturated":              # opaque, large splats: most pixels stop early (T < 1e-4)
        sc["opacities"][0::3] = 1.0
        sc["opacities"][1::3] = 1e-5
        sc["scales"] *= 3.0
    return sc


def _raw_activations(sc):
    """The raw network outputs whose activations are sc's opacities / scales / rotations (up to rounding)."""
    out = dict(sc)
    out["opacities"] = torch.logit(sc["opacities"].clamp(1e-6, 1 - 1e-6))
    out["scales"] = torch.log(sc["scales"])
    out["rotations"] = sc["rotations"] * 1.7
    return out


def _both(fn):
    """fn(for_backward) for the training forward and the forward-only one, after a synchronise each."""
    a = fn(True)
    torch.cuda.synchronize()
    b = fn(False)
    torch.cuda.synchronize()
    return a, b


def _same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    assert torch.equal(a, b), f"{what}: {(a != b).sum().item()} elements differ"


def _transmats(scd, st, P, H, W):
    from lara_b200 import rasterizer as R
    from lara_b200.debug import unpack_state
    _, _, r0, s0 = R.forward_raw(scd["means3D"], scd["shs"], None, scd["opacities"], scd["scales"], scd["rotations"],
                                 None, st)
    torch.cuda.synchronize()
    T = unpack_state(s0, P, H, W)["transMat"].contiguous().clone()
    T[r0 <= 0] = 0
    return T


@pytest.mark.parametrize("P,H,W,deg,variant", [
    (20000, 128, 128, 0, "sh"), (20000, 128, 128, 1, "sh"), (20000, 128, 128, 2, "sh"), (20000, 128, 128, 3, "sh"),
    (20000, 128, 128, 1, "raw"), (20000, 128, 128, 3, "raw"), (20000, 128, 128, 1, "colors_precomp"),
    (20000, 128, 128, 1, "transmat"), (30000, 300, 500, 2, "sh"), (30000, 301, 197, 1, "raw"),
    (8000, 128, 128, 1, "saturated"), (0, 64, 96, 1, "sh"), (131072, 512, 512, 1, "sh"), (131072, 512, 512, 1, "raw"),
])
def test_forward_only_raw_is_bit_identical(cuda_device, P, H, W, deg, variant):
    from lara_b200 import rasterizer as R, scene as S
    dev = cuda_device
    sc = _scene(P, deg, 11, "saturated" if variant == "saturated" else "lara")
    raw = variant == "raw"
    scd = to_dev(_raw_activations(sc) if raw else sc, dev)
    st = S.settings_for(S.cameras(1, H, W, 5)[0], torch.full((3,), 0.3), deg, dev, R.GaussianRasterizationSettings)
    shs, colors, scales, rots, T = scd["shs"], None, scd["scales"], scd["rotations"], None
    if variant == "colors_precomp":
        shs, colors = None, torch.rand((P, 3), generator=torch.Generator().manual_seed(3)).to(dev)
    if variant == "transmat":
        T = _transmats(scd, st, P, H, W)
        scales = rots = None
    a, b = _both(lambda fb: R.forward_raw(scd["means3D"], shs, colors, scd["opacities"], scales, rots, T, st,
                                          raw_activations=raw, for_backward=fb))
    for k, x, y in zip(("color", "allmap", "radii"), a[:3], b[:3]):
        _same(x, y, k)
    assert a[3].num_rendered == b[3].num_rendered
    assert b[3].image is None and b[3].point_list is None and not b[3].for_backward
    if P > 0:
        assert a[2].gt(0).any() and a[1][1].gt(0).any()          # something was rendered
        assert b[3].capacity == a[3].capacity


def _grad_inputs(scd, requires):
    return {k: (v.detach().clone().requires_grad_(True) if requires and k in KEYS else v) for k, v in scd.items()}


@pytest.mark.parametrize("raw", [False, True])
@pytest.mark.parametrize("mode", ["no_grad", "inference_mode", "no_requires_grad"])
def test_dropin_wrappers_take_the_forward_only_path_bit_identically(cuda_device, raw, mode):
    from lara_b200 import _lib, rasterizer as R, scene as S
    dev = cuda_device
    P, H, W, deg = 40000, 200, 232, 2
    sc = _scene(P, deg, 12)
    scd = to_dev(_raw_activations(sc) if raw else sc, dev)
    st = S.settings_for(S.cameras(1, H, W, 6)[0], torch.ones(3), deg, dev, R.GaussianRasterizationSettings)
    rast = R.GaussianRasterizer(st)

    def call(t, m2d):
        if raw:
            return rast.forward_raw_activations(t["means3D"], m2d, t["opacities"], t["scales"], t["rotations"],
                                                shs=t["shs"])
        return rast(means3D=t["means3D"], means2D=m2d, shs=t["shs"], opacities=t["opacities"], scales=t["scales"],
                    rotations=t["rotations"])

    t = _grad_inputs(scd, True)
    m2d = torch.zeros_like(scd["means3D"], requires_grad=True)
    ref = call(t, m2d)
    assert ref[0].grad_fn is not None
    torch.cuda.synchronize()
    _lib.profile_begin()
    if mode == "no_grad":
        with torch.no_grad():
            out = call(t, m2d)
    elif mode == "inference_mode":
        with torch.inference_mode():
            out = call(t, m2d)
    else:
        out = call(scd, torch.zeros_like(scd["means3D"]))
    torch.cuda.synchronize()
    prof = _lib.profile_end()
    assert prof["render_fwd"][1] == 1 and prof["render_bwd"][1] == 0, prof
    for k, x, y in zip(("color", "radii", "allmap"), ref, out):
        _same(x.detach(), y, k)
        assert not y.requires_grad and y.grad_fn is None


def _lara_rays(V, H, W, seed, dev):
    g = torch.Generator().manual_seed(seed)
    return torch.cat([torch.randn((V, H, W, 3), generator=g) * 0.01 + torch.tensor([0.0, 0.0, -1.9]),
                      torch.nn.functional.normalize(torch.randn((V, H, W, 3), generator=g), dim=-1)], -1).to(dev)


@pytest.mark.parametrize("P,H,W,V,deg,raw,rays", [
    (131072, 512, 512, 8, 1, True, True), (131072, 512, 512, 8, 1, False, True), (50000, 201, 333, 8, 3, True, True),
    (50000, 256, 256, 3, 0, True, False), (0, 64, 64, 4, 1, True, True),
])
def test_render_scene_views_forward_only_is_bit_identical(cuda_device, P, H, W, V, deg, raw, rays):
    from lara_b200 import _lib, rasterizer as R, scene as S
    from lara_b200.multiview import render_scene_views
    dev = cuda_device
    sc = _scene(P, deg, 13)
    scd = to_dev(_raw_activations(sc) if raw else sc, dev)
    sets = [S.settings_for(c, torch.full((3,), float(j % 2)), deg, dev, R.GaussianRasterizationSettings)
            for j, c in enumerate(S.cameras(V, H, W, 7))]
    ry = _lara_rays(V, H, W, 8, dev) if rays else None

    def call(t):
        return render_scene_views(t["means3D"], t["shs"], t["opacities"], t["scales"], t["rotations"], sets, rays=ry,
                                  depth_ratio=0.3, raw_activations=raw)

    t = _grad_inputs(scd, True)
    ref = call(t)
    torch.cuda.synchronize()
    _lib.profile_begin()
    with torch.no_grad():
        out = call(t)
    torch.cuda.synchronize()
    prof = _lib.profile_end()
    assert prof["render_fwd"][1] == (1 if P > 0 else 0) and prof["render_bwd"][1] == 0, prof
    with torch.inference_mode():
        out2 = call(t)
    torch.cuda.synchronize()
    assert set(ref) == set(out) == set(out2)
    for k in ref:
        _same(ref[k].detach(), out[k], k)
        _same(ref[k].detach(), out2[k], k)
        assert ref[k].stride() == out[k].stride(), k


def test_forward_only_overflow_repairs_itself_like_the_training_forward(cuda_device, monkeypatch):
    from lara_b200 import rasterizer as R, scene as S
    dev = cuda_device
    P, H, W, V = 60000, 256, 256, 3
    scd = to_dev(_scene(P, 1, 14), dev)
    sets = [S.settings_for(c, torch.ones(3), 1, dev, R.GaussianRasterizationSettings) for c in S.cameras(V, H, W, 9)]
    cams = R.pack_cameras(sets, dev)
    monkeypatch.setattr(R, "initial_capacity", lambda P, device: 4096)
    outs = []
    for fb in (True, False):
        color, allmap, radii, state = R.forward_views_raw(scd["means3D"], scd["shs"], None, scd["opacities"],
                                                          scd["scales"], scd["rotations"], None, cams, sets[0].tanfovx,
                                                          sets[0].tanfovy, H, W, 1, for_backward=fb)
        with pytest.warns(RuntimeWarning, match="exceeded the optimistic capacity"):
            counts = state.resolve()
        assert max(counts) > 4096 and state.capacity > max(counts)
        assert (state.point_list is not None) == fb
        torch.cuda.synchronize()
        outs.append((color, allmap, radii, counts))
    for k, x, y in zip(("color", "allmap", "radii", "counts"), *outs):
        if k == "counts":
            assert x == y
        else:
            _same(x, y, k)


def _peak_and_left(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    color, allmap, radii, state = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    capacity = state.capacity
    state.resolve()
    del state
    left = torch.cuda.memory_allocated() - base
    outputs = sum((t.numel() * t.element_size() + 511) // 512 * 512 for t in (color, allmap, radii))
    return peak, left, outputs, capacity


def test_forward_only_needs_the_record_bytes_less_memory(cuda_device):
    """One call at 131 072 Gaussians, 512 x 512, 8 views: the forward-only peak is below the training forward's by at
    least the contribution record (32 B per instance of capacity and view) less 8 MiB of allocator rounding; after the
    call and its count read-back only the outputs stay allocated (within 4 MiB of rounding)."""
    from lara_b200 import rasterizer as R, scene as S
    dev = cuda_device
    P, H, W, V = 131072, 512, 512, 8
    scd = to_dev(_scene(P, 1, 15), dev)
    sets = [S.settings_for(c, torch.ones(3), 1, dev, R.GaussianRasterizationSettings) for c in S.cameras(V, H, W, 10)]
    cams = R.pack_cameras(sets, dev)

    def run(fb):
        return lambda: R.forward_views_raw(scd["means3D"], scd["shs"], None, scd["opacities"], scd["scales"],
                                           scd["rotations"], None, cams, sets[0].tanfovx, sets[0].tanfovy, H, W, 1,
                                           for_backward=fb)

    run(True)()                  # settle the capacity high-water mark, so both calls get the same capacity
    torch.cuda.synchronize()
    R._drain_ready(dev)
    peak_t, left_t, out_t, cap_t = _peak_and_left(run(True))
    peak_f, left_f, out_f, cap_f = _peak_and_left(run(False))
    assert cap_t == cap_f
    record = 8 * 4 * cap_f * V
    assert peak_t - peak_f >= record - (8 << 20), (peak_t, peak_f, record)
    assert out_f == out_t and out_f <= left_f <= out_f + (4 << 20), (left_f, out_f)


def test_forward_only_call_between_a_forward_and_its_backward_changes_no_gradient_bit(cuda_device):
    """Deterministic backward: a training forward, then a forward-only render of another scene, then the training
    forward's backward gives the same gradient bits as without the render in between."""
    from lara_b200 import rasterizer as R, scene as S
    dev = cuda_device
    P, H, W, V = 60000, 256, 256, 4
    scd = to_dev(_scene(P, 1, 16), dev)
    other = to_dev(_scene(P, 1, 17), dev)
    sets = [S.settings_for(c, torch.ones(3), 1, dev, R.GaussianRasterizationSettings) for c in S.cameras(V, H, W, 11)]
    cams = R.pack_cameras(sets, dev)
    ups = [torch.stack([S.upstream_grads(H, W, 20 + v)[i] for v in range(V)]).to(dev).contiguous() for i in range(2)]
    args = (None, cams, sets[0].tanfovx, sets[0].tanfovy, H, W, 1)

    def fwd(s, fb):
        return R.forward_views_raw(s["means3D"], s["shs"], None, s["opacities"], s["scales"], s["rotations"], *args,
                                   for_backward=fb)

    def bwd(radii, state):
        g = R.backward_views_raw(state, radii, scd["means3D"], scd["shs"], None, scd["scales"], scd["rotations"], None,
                                 cams, sets[0].tanfovx, sets[0].tanfovy, H, W, 1, ups[0], ups[1], need_means2D=True,
                                 deterministic=True)
        torch.cuda.synchronize()
        return g

    _, _, radii, state = fwd(scd, True)
    g_plain = bwd(radii, state)
    _, _, radii, state = fwd(scd, True)
    c_o, a_o, _, st_o = fwd(other, False)
    g_mixed = bwd(radii, state)
    for k, v in g_plain.items():
        if v is not None:
            _same(v, g_mixed[k], k)
    with pytest.raises(RuntimeError, match="forward-only"):
        bwd(radii, st_o)


class _Cam(NamedTuple):
    image_height: int
    image_width: int
    FoVx: float
    FoVy: float
    world_view_transform: torch.Tensor
    full_proj_transform: torch.Tensor
    camera_center: torch.Tensor


@pytest.mark.parametrize("fused", [True, False])
def test_renderer_under_no_grad_and_inference_mode_matches_grad_mode(cuda_device, fused):
    from lara_b200 import scene as S
    from lara_b200.renderer import Renderer
    dev = cuda_device
    P, H, W, V = 50000, 224, 288, 3
    scd = to_dev(_raw_activations(_scene(P, 3, 18)), dev)      # the Renderer applies the activations either way
    cams = [_Cam(H, W, 2 * math.atan(c.tanfovx), 2 * math.atan(c.tanfovy), c.viewmatrix.to(dev),
                 c.projmatrix.to(dev), c.campos.to(dev)) for c in S.cameras(V, H, W, 12)]
    rays = _lara_rays(V, H, W, 19, dev)
    ren = Renderer(sh_degree=3, white_background=False, fused_activations=fused)

    def run():
        one = ren.render_img(cams[0], rays[0], t["means3D"], t["shs"], t["opacities"], t["scales"], t["rotations"],
                             dev, depth_ratio=0.2)
        plain = ren.render_img(cams[1], None, t["means3D"], t["shs"], t["opacities"], t["scales"], t["rotations"], dev)
        views = ren.render_views(cams, rays, t["means3D"], t["shs"], t["opacities"], t["scales"], t["rotations"], dev,
                                 depth_ratio=0.2)
        return {**{"one/" + k: v for k, v in one.items()}, "plain": plain, **{"views/" + k: v for k, v in views.items()}}

    t = _grad_inputs(scd, True)
    ref = run()
    assert ref["one/image"].requires_grad and ref["views/image"].requires_grad
    with torch.no_grad():
        a = run()
    with torch.inference_mode():
        b = run()
    torch.cuda.synchronize()
    for k in ref:
        _same(ref[k].detach(), a[k], k)
        _same(ref[k].detach(), b[k], k)
        assert not a[k].requires_grad and not b[k].requires_grad


def test_forward_only_scene_views_launch_no_backward_kernel_and_warn_nothing(cuda_device):
    """A forward-only render_scene_views issues one launch per kernel and none of the backward's."""
    from lara_b200 import _lib, rasterizer as R, scene as S
    from lara_b200.multiview import render_scene_views
    dev = cuda_device
    P, H, W, V = 30000, 256, 256, 6
    scd = to_dev(_scene(P, 1, 19), dev)
    sets = [S.settings_for(c, torch.ones(3), 1, dev, R.GaussianRasterizationSettings) for c in S.cameras(V, H, W, 13)]
    render_scene_views(scd["means3D"], scd["shs"], scd["opacities"], scd["scales"], scd["rotations"], sets)
    torch.cuda.synchronize()
    for _ in range(3):
        _lib.profile_begin()
        with warnings.catch_warnings():
            warnings.simplefilter("error")
            with torch.no_grad():
                render_scene_views(scd["means3D"], scd["shs"], scd["opacities"], scd["scales"], scd["rotations"], sets)
            torch.cuda.synchronize()
        prof = _lib.profile_end()
        assert prof["render_fwd"][1] == 1 and prof["render_bwd"][1] == 0 and prof["preprocess_bwd"][1] == 0, prof
        assert all(n <= 1 for _, n in prof.values()), prof
