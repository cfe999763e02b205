"""Deterministic gradients (DESIGN §3.13): with torch.use_deterministic_algorithms(True) the blend backward, the
point-feature backward and the loss sums add their terms in an order-independent way, so two identical steps give
bit-identical results.

* CPU: the fixed-point helpers of csrc/det_sum.cuh, built for the host, against math.fsum -- the same bits under any
  order of the terms, the stated error bound, and the overflow guard at exactly its budget; the resolution of the
  deterministic flag.
* GPU: repeatability of every returned gradient with unrelated work enqueued between two runs; the per-Gaussian
  float64 replay of tests/test_grad_per_gaussian.py in deterministic mode; the point features and the loss; the fused
  LaRa chain end to end; the overflow guard.
"""
import contextlib
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "lara_b200", "csrc")

_HOST_SRC = r"""
#include "det_sum.cuh"
using namespace srf::det;
extern "C" {
int h_scale_exp(uint32_t bits, int L) { return scale_exp(bits, L); }
int h_quantize(float x, int k, int L, long long* q) { return quantize(x, k, L, *q) ? 1 : 0; }
float h_to_float(long long S, int k) { return to_float(S, k); }
// the whole scheme over n terms in the given order: bound, count, scale, quantise, wrapping sum, convert
int h_sum(const float* x, int n, float* out, int* k_out) {
    uint32_t b = 0;
    for (int i = 0; i < n; ++i) b = abs_bits(x[i]) > b ? abs_bits(x[i]) : b;
    const int L = ceil_log2((uint64_t)n), k = scale_exp(b, L);
    unsigned long long S = 0;
    int ok = 1;
    for (int i = 0; i < n; ++i) {
        long long q;
        ok &= quantize(x[i], k, L, q) ? 1 : 0;
        S += (unsigned long long)q;
    }
    *out = to_float((long long)S, k);
    *k_out = k;
    return ok;
}
}
"""


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    d = tmp_path_factory.mktemp("det_sum")
    src, so = d / "det_sum_host.cpp", d / "libdet_sum_host.so"
    src.write_text(_HOST_SRC)
    subprocess.run(["c++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-I", CSRC, str(src), "-o",
                    str(so)], check=True, timeout=300)
    lib = ctypes.CDLL(str(so))
    lib.h_scale_exp.argtypes, lib.h_scale_exp.restype = [ctypes.c_uint32, ctypes.c_int], ctypes.c_int
    lib.h_quantize.argtypes = [ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_longlong)]
    lib.h_to_float.argtypes, lib.h_to_float.restype = [ctypes.c_longlong, ctypes.c_int], ctypes.c_float
    lib.h_sum.argtypes = [ctypes.POINTER(ctypes.c_float), ctypes.c_int, ctypes.POINTER(ctypes.c_float),
                          ctypes.POINTER(ctypes.c_int)]
    return lib


def _sum(host, x):
    x = np.ascontiguousarray(x, dtype=np.float32)
    out, k = ctypes.c_float(), ctypes.c_int()
    ok = host.h_sum(x.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), len(x), ctypes.byref(out), ctypes.byref(k))
    return bool(ok), np.float32(out.value), k.value


def _spread(rng, n, emin, emax):
    """n fp32 values with random signs, mantissas and binary exponents uniform in [emin, emax]."""
    v = rng.uniform(1.0, 2.0, n) * np.exp2(rng.integers(emin, emax + 1, n).astype(np.float64))
    return (v * rng.choice([-1.0, 1.0], n)).astype(np.float32)


@pytest.mark.parametrize("n,emin,emax,seed", [(1, -20, 20, 0), (7, -149, -120, 1), (1000, -60, 60, 2),
                                              (4097, -149, 127, 3), (20000, -10, 10, 4), (300, 100, 126, 5)])
def test_fixed_point_sum_is_order_independent_and_within_its_bound(host, n, emin, emax, seed):
    rng = np.random.default_rng(seed)
    x = _spread(rng, n, emin, emax)
    ok, ref_bits, k = _sum(host, x)
    assert ok
    for _ in range(12):
        ok2, got, k2 = _sum(host, rng.permutation(x))
        assert ok2 and k2 == k and got.view(np.uint32) == ref_bits.view(np.uint32)
    exact = math.fsum(float(v) for v in x)
    # n half-units of the last fixed-point place, one fp32 rounding of the result, and the subnormal floor
    bound = n * 2.0 ** -(k + 1) + 2.0 ** -24 * abs(float(ref_bits)) + 2.0 ** -150
    assert abs(float(ref_bits) - exact) <= bound, (float(ref_bits), exact, bound)
    # the bound is the documented one: n^2 m 2^-61 for the quantisation part
    m = float(np.abs(x).max())
    assert n * 2.0 ** -(k + 1) <= n * n * m * 2.0 ** -61 * 2


def test_fixed_point_sum_of_terms_at_the_bound_is_exact(host):
    """2^L terms all equal to the bound: the largest sum the scale admits, exact and without overflow."""
    for L, m in ((0, 3.0e38), (5, 1.7e38), (12, 1.0e-30), (16, 1e-45), (20, 0.75)):
        x = np.full(1 << L, m, np.float32)
        ok, got, k = _sum(host, x)
        assert ok
        with np.errstate(over="ignore"):
            want = np.float32(float(np.float32(m)) * (1 << L))       # inf past the fp32 range, as the sum's rounding
        assert got == want, (L, m, got, want)
        ok, got_neg, _ = _sum(host, -x)
        assert ok and float(got_neg) == -float(got)


def test_overflow_guard_fires_exactly_past_the_budget(host):
    q = ctypes.c_longlong()
    for L, k in ((0, 0), (3, 10), (20, -30), (40, 100), (60, 150)):
        lim = np.float32(2.0 ** (62 - L - k))         # |x 2^k| == 2^(62-L): the largest accepted term
        assert host.h_quantize(lim, k, L, ctypes.byref(q)) == 1 and q.value == 1 << (62 - L)
        assert host.h_quantize(-lim, k, L, ctypes.byref(q)) == 1 and q.value == -(1 << (62 - L))
        above = np.nextafter(lim, np.float32(np.inf))
        assert host.h_quantize(above, k, L, ctypes.byref(q)) == 0 and q.value == 0
        assert host.h_quantize(-above, k, L, ctypes.byref(q)) == 0
    for bad in (np.inf, -np.inf, np.nan):
        assert host.h_quantize(np.float32(bad), 0, 0, ctypes.byref(q)) == 0
        ok, _, _ = _sum(host, np.array([1.0, bad, 2.0], np.float32))
        assert not ok
    # a bound taken from the terms never lets one of them fail, including the 2x margin's neighbours
    for bits in (0x00000001, 0x007fffff, 0x00800000, 0x3f800000, 0x7f7fffff):
        for L in (0, 7, 33):
            k = host.h_scale_exp(bits, L)
            m = np.array([bits], np.uint32).view(np.float32)[0]
            with np.errstate(over="ignore"):
                near = [x for x in (m, np.nextafter(m, np.float32(np.inf)), np.float32(2 * float(m))) if np.isfinite(x)]
            for x in near:
                assert host.h_quantize(x, k, L, ctypes.byref(q)) == 1, (hex(bits), L, x)


def test_round_trip_and_scale_range(host):
    for k in (-132, -40, 0, 77, 186):
        for S in (0, 1, -1, 123456789, (1 << 62) - 1, -(1 << 62)):
            with np.errstate(over="ignore"):
                want = np.float32(float(np.float32(float(S))) * 2.0 ** -k)
            assert host.h_to_float(S, k) == want
    assert host.h_scale_exp(0, 0) == 186 and host.h_scale_exp(0x7f800000, 64) == -132


def test_flag_resolution():
    from lara_b200._lib import use_deterministic
    for enabled in (False, True):
        for warn in (False, True):
            assert use_deterministic(True, enabled, warn) is True
            assert use_deterministic(False, enabled, warn) is False
            assert use_deterministic(None, enabled, warn) is (enabled or warn)


def test_flag_follows_torch():
    from lara_b200 import _lib
    with _torch_flag(False):
        assert not _lib.deterministic() and _lib.deterministic(True)
    with _torch_flag(True):
        assert _lib.deterministic() and not _lib.deterministic(False)
    with _torch_flag(True, warn_only=True):
        assert _lib.deterministic()


def test_scratch_queries(lib):
    from lara_b200 import _lib
    V, P = 8, 524288
    det = _lib.det_backward_scratch_bytes(lib, V, P)
    default = _lib.views_sizes(lib, V, P, 512, 512, 0)[5]
    assert det >= default + V * P * 224
    assert _lib.det_point_feats_workspace_bytes(lib, 2, 64, 80) >= 5 * 2 * 64 * 80 * 8
    assert _lib.det_loss_workspace_bytes(lib, 8, 512, 512) == 1024 * 24
    n = ctypes.c_size_t()
    assert lib.srf_views_backward_deterministic_scratch_bytes(0, 10, ctypes.byref(n)) != 0
    assert b"deterministic" in lib.srf_last_error()
    assert lib.srf_point_feats_deterministic_workspace_bytes(1, 0, 4, ctypes.byref(n)) != 0
    assert lib.srf_loss_deterministic_workspace_bytes(1, 4, -1, ctypes.byref(n)) != 0


def test_scenes_backward_and_fused_ops_reject_bad_arguments_before_any_launch(lib):
    # null cameras / null input / misaligned workspace: status and message, no CUDA call
    from lara_b200 import _lib
    args = [None, 1, 1, 10, None, 0, 1, 16, 16, 0, None, None, None, 0, None, None, 0, _lib.tan_fov_array([(1.0, 1.0)]),
            None, None, None, None, None, None, None, None, 0, None, None, None, None, None, None, None, None, 0, 1]
    assert lib.srf_scenes_backward(*args) != 0
    assert b"srf_scenes_backward" in lib.srf_last_error()
    assert lib.srf_loss_forward(None, 1, 8, 8, 0, None, 1, None, None, None, None, 1, None) != 0
    assert b"null pointer" in lib.srf_last_error()
    assert lib.srf_loss_forward(None, 1, 8, 8, 0, 1, 1, None, None, None, None, 1, 1) != 0
    assert b"workspace" in lib.srf_last_error()
    assert lib.srf_point_feats_backward(None, 1, 0, 8, 8, None, 1, 1, 1, 1, 1, 1, None, None, None, None, None, 1) != 0
    assert b"workspace" in lib.srf_last_error()


# ---------------------------------------------------------------------------------------------------------- GPU

@contextlib.contextmanager
def _torch_flag(on, warn_only=False):
    prev, prev_w = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on, warn_only=warn_only)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_w)


def _noise(dev):
    """Unrelated work between two runs: other kernels, other allocations, another stream's timing."""
    a = torch.randn((2048, 2048), device=dev)
    for _ in range(3):
        a = (a @ a.T).tanh_()
    torch.empty(64 << 20, dtype=torch.uint8, device=dev).fill_(7)


def _same(a, b, what):
    if a is None or b is None:
        assert a is None and b is None, what
        return
    assert a.shape == b.shape and torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                                              b.view(torch.int32) if b.dtype == torch.float32 else b), what


def _views_case(P, H, W, V, deg, seed, dev):
    from lara_b200 import rasterizer as R
    from lara_b200 import scene as S
    sc = S.scene(P, seed, deg)
    cams = S.cameras(V, H, W, seed)
    bg = torch.tensor([0.3, 0.5, 0.2])
    settings = [S.settings_for(c, bg, deg, dev, R.GaussianRasterizationSettings) for c in cams]
    g = torch.Generator().manual_seed(seed)
    ups = (torch.randn((V, 3, H, W), generator=g) / (H * W), torch.randn((V, 8, H, W), generator=g) / (H * W))
    t = {k: sc[k].to(dev).contiguous() for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    return t, settings, R.pack_cameras(settings, dev), tuple(u.to(dev) for u in ups), cams


def _lists(state, lib, V, P, H, W):
    from lara_b200 import _lib
    counts = state.resolve()
    stride = _lib.views_sizes(lib, V, P, H, W, state.capacity)[4] // V
    return [state.point_list[v * stride: v * stride + 4 * counts[v]].clone() for v in range(V)]


def _views_fwd_bwd(t, cams, tan, ups, H, W, deg, lib, deterministic):
    from lara_b200 import rasterizer as R
    V, P = int(cams.shape[0]), int(t["means3D"].shape[0])
    color, allmap, radii, state = R.forward_views_raw(t["means3D"], t["shs"], None, t["opacities"], t["scales"],
                                                      t["rotations"], None, cams, tan[0], tan[1], H, W, deg)
    g = R.backward_views_raw(state, radii, t["means3D"], t["shs"], None, t["scales"], t["rotations"], None, cams,
                             tan[0], tan[1], H, W, deg, ups[0], ups[1], need_means2D=True, deterministic=deterministic)
    torch.cuda.synchronize()
    return (color, allmap, radii, _lists(state, lib, V, P, H, W)), g


@pytest.mark.gpu
@pytest.mark.parametrize("P,H,W,V,deg", [(131072, 512, 512, 8, 1), (524288, 512, 512, 8, 1), (20000, 200, 312, 3, 0),
                                         (20000, 200, 312, 3, 1), (15000, 130, 170, 2, 2), (15000, 333, 97, 2, 3)])
def test_views_backward_repeats_bit_for_bit(cuda_device, lib, P, H, W, V, deg):
    dev = cuda_device
    t, settings, cams, ups, cs = _views_case(P, H, W, V, deg, P % 97 + deg, dev)
    tan = (cs[0].tanfovx, cs[0].tanfovy)
    f1, g1 = _views_fwd_bwd(t, cams, tan, ups, H, W, deg, lib, True)
    _noise(dev)
    f2, g2 = _views_fwd_bwd(t, cams, tan, ups, H, W, deg, lib, True)
    for a, b, name in zip(f1[:3], f2[:3], ("color", "allmap", "radii")):
        _same(a, b, name)
    for v, (a, b) in enumerate(zip(f1[3], f2[3])):
        _same(a, b, f"point_list of view {v}")
    for k in g1:
        _same(g1[k], g2[k], k)
    # and the deterministic gradients are the default ones up to the default path's own summation noise
    _, gd = _views_fwd_bwd(t, cams, tan, ups, H, W, deg, lib, False)
    for k in ("means3D", "sh", "opacities", "scales", "rotations", "means2D"):
        a, b = g1[k].double(), gd[k].double()
        assert (a - b).abs().max() <= 1e-5 * b.abs().max(), k


def _dropin(sc, cam, dev, deterministic, colors=None, transMat=None, raw=False):
    from lara_b200 import rasterizer as R
    from lara_b200 import scene as S
    st = S.settings_for(cam, torch.tensor([0.2, 0.4, 0.6]), sc["sh_degree"], dev, R.GaussianRasterizationSettings)
    t = lambda k: sc[k].float().to(dev).contiguous()        # noqa: E731
    shs = None if colors is not None else t("shs")
    cols = None if colors is None else colors.to(dev)
    tm = None if transMat is None else transMat.to(dev).contiguous()
    sca, rot = (None, None) if tm is not None else (t("scales"), t("rotations"))
    gc, ga = S.upstream_grads(cam.image_height, cam.image_width, 3)
    color, allmap, radii, state = R.forward_raw(t("means3D"), shs, cols, t("opacities"), sca, rot, tm, st,
                                                raw_activations=raw)
    g = R.backward_raw(state, radii, t("means3D"), shs, cols, sca, rot, tm, st, gc.to(dev), ga.to(dev),
                       raw_activations=raw, deterministic=deterministic)
    torch.cuda.synchronize()
    return g, state


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["sh", "colors_precomp", "transMat_precomp", "raw"])
def test_single_view_backward_repeats_bit_for_bit(cuda_device, mode):
    from lara_b200 import scene as S
    from lara_b200.debug import unpack_state
    dev = cuda_device
    sc = S.scene(30000, 11, 2)
    cam = S.cameras(2, 192, 224, 11)[1]
    kw = {}
    if mode == "colors_precomp":
        kw["colors"] = torch.rand((30000, 3), generator=torch.Generator().manual_seed(1))
    elif mode == "transMat_precomp":
        _, st = _dropin(sc, cam, dev, False)
        kw["transMat"] = unpack_state(st, 30000, 192, 224)["transMat"].float()
    elif mode == "raw":
        o = sc["opacities"]
        sc = dict(sc, opacities=torch.log(o / (1 - o)), scales=torch.log(sc["scales"]), rotations=sc["rotations"] * 2.3)
        kw["raw"] = True
    g1, _ = _dropin(sc, cam, dev, True, **kw)
    _noise(dev)
    g2, _ = _dropin(sc, cam, dev, True, **kw)
    gd, _ = _dropin(sc, cam, dev, False, **kw)
    for k in g1:
        _same(g1[k], g2[k], k)
        if g1[k] is not None:
            assert (g1[k] - gd[k]).abs().max() <= 1e-5 * gd[k].abs().max(), k


@pytest.mark.gpu
def test_drop_in_and_sharded_accumulate_follow_the_torch_flag(cuda_device):
    from lara_b200 import GaussianRasterizationSettings, GaussianRasterizer, _lib
    from lara_b200 import scene as S
    from lara_b200 import sharded
    dev = cuda_device
    sc = S.scene(20000, 12, 1)
    cams = S.cameras(4, 160, 160, 12)
    settings = [S.settings_for(c, torch.ones(3), 1, dev, GaussianRasterizationSettings) for c in cams]
    params = {k: sc[k].to(dev).contiguous() for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    ups = [tuple(u.to(dev) for u in S.upstream_grads(160, 160, v)) for v in range(4)]

    def dropin():
        leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
        m2d = torch.zeros_like(leaves["means3D"], requires_grad=True)
        color, radii, allmap = GaussianRasterizer(settings[0])(
            means3D=leaves["means3D"], means2D=m2d, shs=leaves["shs"], opacities=leaves["opacities"],
            scales=leaves["scales"], rotations=leaves["rotations"])
        torch.autograd.backward((color, allmap), ups[0])
        return [leaves[k].grad for k in params] + [m2d.grad]

    def shard():
        grads = sharded.GradBuffer(20000, 4, dev)
        grads.flat.copy_(torch.randn(grads.flat.shape, generator=torch.Generator().manual_seed(5)).to(dev) * 1e-3)
        sharded.render_views(params, settings, lambda vid, c, a: ups[vid], grads=grads)
        return [grads.flat.clone()]

    for fn in (dropin, shard):
        with _torch_flag(True):
            _lib.profile_begin()
            a = fn()
            prof = _lib.profile_end()
            _noise(dev)
            b = fn()
        assert prof["render_bwd"][1] == 2, prof          # bound pass + fixed-point pass
        for x, y in zip(a, b):
            _same(x, y, fn.__name__)
        _lib.profile_begin()
        fn()
        assert _lib.profile_end()["render_bwd"][1] == 1


# --------------------------------------------------------------------------------------- accuracy (float64 replay)

@pytest.mark.gpu
def test_replay_bound_holds_in_deterministic_mode(cuda_device):
    import test_grad_per_gaussian as T
    from lara_b200 import scene as S
    sc = S.scene(8000, 5)
    cam = S.cameras(3, 128, 144, 5)[0]
    gc, ga = T._upstream(128, 144, 1, None)
    bg = np.array([0.2, 0.5, 0.9], np.float32)
    _, _, worst_default = T._kernel_vs_replay(sc, cam, bg, gc, ga, cuda_device)
    with _torch_flag(True, warn_only=True):
        r, _, worst_det = T._kernel_vs_replay(sc, cam, bg, gc, ga, cuda_device)
    print(f"worst err/bound: deterministic {worst_det:.3g}, default {worst_default:.3g}")
    assert r["pairs"] > 100_000 and worst_det < 1.0


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["test_kernel_gradients_sub_pixel_and_far_splats",
                                  "test_kernel_gradients_at_chunk_boundaries",
                                  "test_kernel_gradients_ragged_and_sh_degrees",
                                  "test_kernel_gradients_colors_and_transmat_precomp",
                                  "test_kernel_gradients_raw_activations",
                                  "test_kernel_gradients_of_three_views_with_accumulate"])
def test_replay_cases_in_deterministic_mode(cuda_device, case):
    """The per-element |kernel - replay| <= bound cases of the default path (low-pass, chunk boundaries, ragged sizes,
    precomputed inputs, raw activations, V = 3 with accumulate), run with the deterministic backward."""
    import test_grad_per_gaussian as T
    fn = getattr(T, case)
    with _torch_flag(True, warn_only=True):
        if case == "test_kernel_gradients_ragged_and_sh_degrees":
            fn(cuda_device, 3)
        else:
            fn(cuda_device)


# ----------------------------------------------------------------------------------------- point features, loss

@pytest.mark.gpu
def test_point_feats_backward_repeats_and_matches_default(cuda_device):
    from test_point_feats import make_case
    from lara_b200.point_feats import sample_point_feats
    dev = cuda_device
    points, img_ref, rend, w2c, ixt = make_case(4, 96, 128, 60000, 3)
    up = torch.randn((4, 8, 60000), generator=torch.Generator().manual_seed(4)).to(dev)

    def run():
        p = points.to(dev).clone().requires_grad_(True)
        r = {k: v.to(dev).clone().requires_grad_(True) for k, v in rend.items()}
        f = sample_point_feats(p, img_ref.to(dev), r, w2c.to(dev), ixt.to(dev))
        f.backward(up)
        torch.cuda.synchronize()
        return [p.grad] + [r[k].grad for k in ("image", "acc_map", "depth")]

    with _torch_flag(True):
        a = run()
        _noise(dev)
        b = run()
    d = run()
    for x, y, z in zip(a, b, d):
        _same(x, y, "point_feats")
        assert (x - z).abs().max() <= 1e-6 * z.abs().max()


@pytest.mark.gpu
def test_loss_sums_repeat_and_match_default(cuda_device):
    from lara_b200.loss import scene_loss
    dev = cuda_device
    g = torch.Generator().manual_seed(9)
    V, H, W = 8, 256, 320
    out = {"image": torch.rand((V, H, W, 3), generator=g), "rend_dist": torch.rand((V, H, W), generator=g) * 0.01,
           "acc_map": torch.rand((V, H, W), generator=g),
           "rend_normal": torch.nn.functional.normalize(torch.rand((V, H, W, 3), generator=g) - 0.5, dim=-1),
           "depth_normal": torch.nn.functional.normalize(torch.rand((V, H, W, 3), generator=g) - 0.5, dim=-1)}
    out = {k: v.to(dev) for k, v in out.items()}
    tar = torch.rand((V, H, W, 3), generator=g).to(dev)
    with _torch_flag(True):
        a = scene_loss(out, tar, 2000)
        _noise(dev)
        b = scene_loss(out, tar, 2000)
    d = scene_loss(out, tar, 2000)
    for k in a[1]:
        _same(a[1][k], b[1][k], k)
        assert (a[1][k] - d[1][k]).abs() <= 1e-6 * d[1][k].abs(), k
    _same(a[0], b[0], "loss")


# --------------------------------------------------------------------------------------------------- end to end

def _lara_chain(dev, V, H, W, seed):
    """gaussians_from_decoder -> render_scene_views -> sample_point_feats -> scene_loss(ms_ssim=True) -> backward;
    returns the gradient wrt the decoder output."""
    from test_point_feats import lara_cameras
    from lara_b200 import GaussianRasterizationSettings, scene as S
    from lara_b200.decoder_layout import gaussians_from_decoder
    from lara_b200.loss import scene_loss
    from lara_b200.multiview import render_scene_views
    from lara_b200.point_feats import sample_point_feats
    g = torch.Generator().manual_seed(seed)
    N, K, sh_dim = 16384, 2, 12
    feats = (torch.randn((1, N, K * (10 + sh_dim)), generator=g) * 0.5).to(dev).requires_grad_(True)
    grid = ((torch.rand((N, 3), generator=g) - 0.5) * 0.8).to(dev)
    cams, w2c, ixt = lara_cameras(V, H, W, seed)
    settings = [S.settings_for(c, torch.zeros(3), 1, dev, GaussianRasterizationSettings) for c in cams]
    rays = torch.cat([torch.randn((V, H, W, 3), generator=g) * 0.01 + torch.tensor([0.0, 0.0, -1.9]),
                      torch.nn.functional.normalize(torch.randn((V, H, W, 3), generator=g), dim=-1)], -1).to(dev)
    tar = torch.rand((V, H, W, 3), generator=g).to(dev)
    img_ref = torch.rand((V, 3, H, W), generator=g).to(dev)
    centers, shs, scaling, rotation, opacity = gaussians_from_decoder(feats, grid, K, sh_dim, -2.1792, -4.2, 0.025)
    out = render_scene_views(centers[0], shs[0], opacity[0], scaling[0], rotation[0], settings, rays=rays,
                             raw_activations=True)
    pf = sample_point_feats(centers[0][::7], img_ref, out, w2c.to(dev), ixt.to(dev))
    loss, _ = scene_loss(out, tar, 2000, ms_ssim=True)
    (loss + pf.square().mean()).backward()
    torch.cuda.synchronize()
    return feats.grad


@pytest.mark.gpu
def test_lara_chain_end_to_end_is_bit_reproducible(cuda_device):
    from lara_b200 import _lib
    dev = cuda_device
    with _torch_flag(True):
        _lib.profile_begin()
        a = _lara_chain(dev, 4, 176, 192, 21)
        on = _lib.profile_end()
        _noise(dev)
        b = _lara_chain(dev, 4, 176, 192, 21)
    _same(a, b, "dL/d(decoder output)")
    assert a.abs().max() > 0
    _lib.profile_begin()
    d = _lara_chain(dev, 4, 176, 192, 21)
    off = _lib.profile_end()
    assert on["render_bwd"][1] == 2 and off["render_bwd"][1] == 1, (on, off)
    assert (a - d).abs().max() <= 1e-5 * d.abs().max()


# -------------------------------------------------------------------------------------------------------- guard

@pytest.mark.gpu
@pytest.mark.parametrize("scale", [1e30, 3e38])
def test_huge_upstream_gives_correct_gradients_or_an_error(cuda_device, lib, scale):
    dev = cuda_device
    P, H, W, V = 20000, 160, 160, 2
    t, settings, cams, ups, cs = _views_case(P, H, W, V, 1, 13, dev)
    tan = (cs[0].tanfovx, cs[0].tanfovy)
    ups = (ups[0] * (scale * H * W), ups[1] * (scale * H * W))
    _, gd = _views_fwd_bwd(t, cams, tan, ups, H, W, 1, lib, False)
    try:
        _, g = _views_fwd_bwd(t, cams, tan, ups, H, W, 1, lib, True)
    except RuntimeError as e:
        assert "fixed-point" in str(e)
        return
    for k in ("means3D", "sh", "opacities", "scales", "rotations"):
        ok = torch.isfinite(gd[k])
        assert torch.isfinite(g[k][ok]).all(), k
        assert (g[k][ok].double() - gd[k][ok].double()).abs().max() <= 1e-5 * gd[k][ok].double().abs().max(), k
