"""The fused MS-SSIM term (csrc/ms_ssim.cu) element by element against float64, level by level.

``oracle.ms_ssim64`` restates the kernels' formulas in float64 with a bound per element on what their fp32 evaluation
may differ by (its docstring derives the rules).  So the border pixels a single window reaches through its edge tap,
the seam columns between views and everything levels 3-4 contribute are each held to their own bound, not to a
fraction of the largest gradient.  The kernels' intermediate state -- the pooled pyramid, the fp64 means, the per-plane
values and coefficients, the gradient pyramid -- is read from the workspace (``lara_b200.debug.unpack_ms_ssim``) and
checked link by link on the kernels' own fp32 inputs, so an error inside one level that the other levels would hide
shows where it is made.

CPU part: the statement in float64 equals the independent NumPy/SciPy statement of test_ms_ssim.py; an fp32 NumPy
emulation of the kernels' sequence lies within the bound at every element; the workspace layout query.  GPU part: the
kernels, end to end and link by link.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ms_ssim64 as M
from oracle.oracle import EB
from test_chain_per_element import _pin64, _tightness
from test_ms_ssim import _fspecial_gauss_1d, np_ms_ssim, smooth_pair

f64 = np.float64


def _np_views_cat(a):
    """[V,C,H,W] -> [1,C,H,V*W]: the views side by side."""
    return np.concatenate(list(a), axis=-1)[None]


def _ratio(got, ref: EB, ctx):
    """|got - ref| <= bound at every element; the worst err/bound."""
    a = np.asarray(got, f64).reshape(ref.v.shape)
    err = np.abs(a - ref.v)
    bad = ~(err <= ref.e)
    if bad.any():
        i = tuple(int(j) for j in np.argwhere(bad)[0])
        raise AssertionError(f"{ctx}: {int(bad.sum())} of {bad.size} elements outside their bound, first at {i}: "
                             f"got {a[i]!r}, float64 {ref.v[i]!r}, bound {ref.e[i]!r}")
    with np.errstate(invalid="ignore", divide="ignore"):
        return float(np.where(err > 0, err / ref.e, 0.0).max()) if err.size else 0.0


def _scalar(got, ve, ctx):
    v, e = ve
    assert abs(float(got) - v) <= e, f"{ctx}: {float(got)!r} vs {v!r} +- {e!r}"
    return abs(float(got) - v) / e if e > 0 else 0.0


# ---------------------------------------------------------------------------------------------------------------- CPU

def test_window_is_the_librarys_bit_for_bit():
    assert np.array_equal(M.window(), _fspecial_gauss_1d(11, 1.5).reshape(-1).numpy())


def _cpu_case(case, seed):
    if case == "177x211":
        X, Y = smooth_pair(2, 3, 177, 211, seed, dtype=torch.float32)
        return X.numpy(), Y.numpy()
    xv, yv = smooth_pair(3, 3, 181, 67, seed, dtype=torch.float32)
    return _np_views_cat(xv.numpy()), _np_views_cat(yv.numpy())


@pytest.mark.parametrize("case", ["177x211", "3 views of 181x67"])
@pytest.mark.parametrize("size_average", [True, False])
def test_statement_equals_numpy_statement_float64(case, size_average):
    """Value, level means and gradient of the statement (upstream 1) equal np_ms_ssim to 1e-12 plus the statement's
    bound with double's rounding in place of fp32's."""
    X, Y = _cpu_case(case, 1)
    st = M.ms_ssim64(X, Y, 1.0, size_average)
    nv, ng, nm = np_ms_ssim(X.astype(f64), Y.astype(f64), M.window(), 1.0, size_average)
    nv = np.atleast_1d(nv)
    for i, (v, e) in enumerate(st["out"]):
        _pin64(nv[i], EB(v, e), f"value {i}")
    for (b, c), p in st["planes"].items():
        assert p["state"] == "pos"
        _pin64(nm[:, b, c], EB([m[0] for m in p["m"]], [m[1] for m in p["m"]]), f"means {b, c}")
        _pin64(ng[b, c], p["dX"][0], f"gradient {b, c}")


def _state_of(res, B, C):
    """A link-by-link state ({"X", "Y", "dX", "mean", "coef"}) from an emulation run."""
    pl = res["planes"]
    st = {k: [None] + [np.stack([np.stack([pl[(b, c)][k][l] for c in range(C)]) for b in range(B)])
                       for l in range(1, 5)] for k in ("X", "Y", "dX")}
    for k, key in (("mean", "m"), ("coef", "coef")):
        st[k] = np.array([[[pl[(b, c)][key][l] for c in range(C)] for b in range(B)] for l in range(5)])
    return st


@pytest.mark.parametrize("case", ["177x211", "3 views of 181x67"])
def test_fp32_emulation_within_bound(case):
    """The kernels' sequence in fp32 NumPy (taps in the kernels' order, each fmaf a float64 operation rounded to
    fp32) against both forms of the statement at every element of the pyramid, the maps and every dX_l, and the
    means, values and coefficients; distinct per-batch upstreams."""
    X, Y = _cpu_case(case, 5)
    B, C = X.shape[:2]
    for size_average in (True, False):
        up = np.array([-0.75], np.float32) if size_average else np.array([0.5, -1.25, 2.0][:B], np.float32)
        em = M.ms_ssim64(X, Y, 1.0, size_average, up, arith=M.F32, keep_maps=True)
        e2e = M.ms_ssim64(X, Y, 1.0, size_average, up, keep_maps=True)
        link = M.ms_ssim64(X, Y, 1.0, size_average, up, state=_state_of(em, B, C))
        worst = {}
        for form, st in (("end to end", e2e), ("link", link)):
            w = 0.0
            for key, p in st["planes"].items():
                q = em["planes"][key]
                assert p["state"] == "pos", (form, key)
                for l in range(5):
                    ctx = f"{form} {key} level {l}"
                    w = max(w, _ratio(q["X"][l], p["X"][l], ctx + " X"), _ratio(q["Y"][l], p["Y"][l], ctx + " Y"),
                            _ratio(q["dX"][l], p["dX"][l], ctx + " dX"), _scalar(q["m"][l], p["m"][l], ctx + " mean"),
                            _scalar(q["coef"][l], p["coef"][l], ctx + " coef"))
                    if p["maps"][l] is not None:
                        w = max(w, _ratio(q["maps"][l], p["maps"][l], ctx + " map"))
                w = max(w, _scalar(q["val"], p["val"], f"{form} {key} value"))
            for i, ve in enumerate(st["out"]):
                w = max(w, _scalar(em["out"][i], ve, f"{form} out {i}"))
            worst[form] = w
        p0 = e2e["planes"][(0, 0)]
        print(f"\n{case} size_average={size_average}: fp32 emulation worst err/bound {worst}")
        _tightness("level-0 cs map", p0["maps"][0])
        _tightness("dX_0 end to end", p0["dX"][0])
        _tightness("dX_0 link", link["planes"][(0, 0)]["dX"][0])


LAYOUT_SHAPES = [(1, 3, 512, 4096), (1, 3, 177, 211), (2, 3, 193, 225), (1, 3, 161, 176), (3, 3, 200, 232),
                 (1, 3, 181, 201), (1, 3, 165, 175)]


@pytest.mark.parametrize("B,C,H,W", LAYOUT_SHAPES)
def test_workspace_layout_query(lib, B, C, H, W):
    from lara_b200 import _lib
    L = _lib.ms_ssim_layout(lib, B, C, H, W)
    n = ctypes.c_size_t()
    assert lib.srf_ms_ssim_workspace_bytes(B, C, H, W, ctypes.byref(n)) == 0
    assert L["total"] == n.value
    regions = [L[k] for k in ("pyr", "gpyr", "part", "mean", "val", "coef", "total")]
    assert all(o % 256 == 0 for o in regions) and regions == sorted(regions)
    P = B * C
    x = torch.zeros(1, 1, H, W)
    npyr = ngp = npart = 0
    for l in range(5):
        h, w = x.shape[-2:]
        assert (L["h"][l], L["w"][l]) == (h, w), l
        pad = (h % 2, w % 2) if l < 4 else (0, 0)
        assert (L["py"][l], L["px"][l]) == pad
        assert (L["ntx"][l], L["nty"][l]) == (-(-(w + pad[1]) // 32), -(-(h + pad[0]) // 16))
        assert L["part_l"][l] == npart
        npart += P * L["ntx"][l] * L["nty"][l]
        if l:
            assert (L["pyr_l"][l], L["gpyr_l"][l]) == (npyr, ngp)
            npyr, ngp = npyr + 2 * P * h * w, ngp + P * h * w
        x = F.avg_pool2d(x, 2, padding=[s % 2 for s in x.shape[-2:]])
    assert L["gpyr"] >= 4 * npyr and L["part"] - L["gpyr"] >= 4 * ngp and L["mean"] - L["part"] >= 8 * npart
    assert L["val"] - L["mean"] >= 8 * 5 * P and L["coef"] - L["val"] >= 8 * P and L["total"] - L["coef"] >= 4 * 5 * P
    assert lib.srf_ms_ssim_workspace_layout(B, C, 160, W, (ctypes.c_size_t * 7)(), (ctypes.c_size_t * 15)(),
                                            (ctypes.c_int * 30)()) != 0


# ---------------------------------------------------------------------------------------------------------------- GPU

def _run(X, Y, views, data_range, size_average, upstream):
    """srf_ms_ssim_forward / _backward as lara_b200.ssim._MsSsim calls them, with a workspace the test keeps."""
    from lara_b200 import _lib
    from lara_b200.rasterizer import _raw_stream
    from lara_b200.ssim import _addr, _logical_shape
    lib = _lib.load()
    dev = X.device
    B, C, H, W = _logical_shape(X, views)
    n = ctypes.c_size_t()
    _lib.check(lib.srf_ms_ssim_workspace_bytes(B, C, H, W, ctypes.byref(n)), lib)
    ws = torch.empty(n.value, dtype=torch.uint8, device=dev)
    out = torch.empty(1 if size_average else B, dtype=torch.float32, device=dev)
    ax, ay = _addr(X, views), _addr(Y, views)
    _lib.check(lib.srf_ms_ssim_forward(_raw_stream(dev), B, C, H, W, X.data_ptr(), ctypes.byref(ax), Y.data_ptr(),
                                       ctypes.byref(ay), float(data_range), int(size_average), ws.data_ptr(),
                                       out.data_ptr()), lib)
    up = torch.as_tensor(np.asarray(upstream, np.float32)).to(dev)
    gX = torch.empty_like(X)
    ag = _addr(gX, views)
    _lib.check(lib.srf_ms_ssim_backward(_raw_stream(dev), B, C, H, W, X.data_ptr(), ctypes.byref(ax), Y.data_ptr(),
                                        ctypes.byref(ay), float(data_range), int(size_average), ws.data_ptr(),
                                        up.data_ptr(), gX.data_ptr(), ctypes.byref(ag)), lib)
    torch.cuda.synchronize()
    return out, gX, ws, (B, C, H, W)


def _logical(t, views):
    a = t.detach().cpu().numpy()
    return _np_views_cat(a) if views else a


def check_kernels(X, Y, views, data_range, size_average, upstream, ctx):
    """Run the kernels and hold every element to the statement, end to end and link by link.  Returns the worst
    err/bound per form."""
    from lara_b200.debug import unpack_ms_ssim
    out, gX, ws, (B, C, H, W) = _run(X, Y, views, data_range, size_average, upstream)
    u = unpack_ms_ssim(ws, B, C, H, W)
    st = {k: [None if a is None else a.cpu().numpy() for a in u[k]] for k in ("X", "Y", "dX")}
    st.update(mean=u["mean"].cpu().numpy(), coef=u["coef"].cpu().numpy())
    val = u["val"].cpu().numpy()
    x, y, g0, o = _logical(X, views), _logical(Y, views), _logical(gX, views), out.cpu().numpy()
    worst = {}
    for form in ("end to end", "link"):
        res = M.ms_ssim64(x, y, data_range, size_average, upstream, state=st if form == "link" else None)
        w = 0.0
        for (b, c), p in res["planes"].items():
            assert p["state"] == "pos", f"{ctx}: plane {b, c} is {p['state']}, means {p['m']}"
            pc = f"{ctx} {form} plane {b, c}"
            for l in range(5):
                if l:
                    w = max(w, _ratio(st["X"][l][b, c], p["X"][l], f"{pc} X_{l}"),
                            _ratio(st["Y"][l][b, c], p["Y"][l], f"{pc} Y_{l}"),
                            _ratio(st["dX"][l][b, c], p["dX"][l], f"{pc} dX_{l}"))
                w = max(w, _scalar(st["mean"][l, b, c], p["m"][l], f"{pc} mean {l}"),
                        _scalar(st["coef"][l, b, c], p["coef"][l], f"{pc} coef {l}"))
            w = max(w, _scalar(val[b, c], p["val"], f"{pc} value"),
                    _ratio(g0[b, c], p["dX"][0], f"{pc} dX_0 (through the addressing record)"))
        for i, ve in enumerate(res["out"]):
            w = max(w, _scalar(o[i], ve, f"{ctx} {form} out {i}"))
        worst[form] = w
        p0 = res["planes"][(0, 0)]
        print(f"\n  {ctx} {form}: worst err/bound {w:.3g}")
        for l in (0, 4):
            _tightness(f"dX_{l}", p0["dX"][l])
        m = p0["m"]
        print(f"  means: bound / value {', '.join(f'{e / v:.2g}' for v, e in m)}; kernel - statement "
              f"{', '.join(f'{st['mean'][l, 0, 0] - m[l][0]:.2g}' for l in range(5))}")
    return worst, out, gX


GPU_CASES = {
    # name: (B, C, H, W, V (views side by side; 0 = one strided image), channel-last, seed, data_range, size_average,
    #        upstream)
    "odd_177x211": (2, 3, 177, 211, 0, False, 12, 1.0, True, [1.0]),
    "tile_edges_193x225": (1, 3, 193, 225, 0, False, 13, 1.0, True, [-0.5]),
    "tile_edges_225x193": (1, 3, 225, 193, 0, True, 14, 1.0, True, [1.0]),
    "min_161x176": (1, 3, 161, 176, 0, False, 15, 1.0, True, [1.0]),
    "min_176x161": (1, 3, 176, 161, 0, False, 16, 1.0, True, [1.0]),
    "odd_views_3x181x67": (1, 3, 181, 67, 3, False, 17, 1.0, True, [-0.5]),
    "odd_views_5x165x35": (1, 3, 165, 35, 5, False, 18, 1.0, True, [-1.0]),
    "per_batch_B3_255": (3, 3, 200, 232, 0, True, 19, 255.0, False, [0.75, -1.5, 2.25]),
}


def _inputs(B, C, H, W, V, channel_last, seed, data_range, dev):
    X, Y = smooth_pair(V or B, C, H, W, seed)
    X, Y = (X * data_range).float(), (Y * data_range).float()
    if channel_last:
        X, Y = (t.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2) for t in (X, Y))
    return X.to(dev), Y.to(dev)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(GPU_CASES))
def test_kernels_per_element(cuda_device, case):
    B, C, H, W, V, cl, seed, R, size_average, up = GPU_CASES[case]
    X, Y = _inputs(B, C, H, W, V, cl, seed, R, cuda_device)
    check_kernels(X, Y, V > 0, R, size_average, up, case)


@pytest.mark.gpu
def test_kernels_per_element_y_equals_x(cuda_device):
    """Y = X: cs = 1 and the gradient cancels to near zero, each element held to its own bound."""
    X, _ = _inputs(1, 3, 183, 197, 0, False, 20, 1.0, cuda_device)
    _, gX = check_kernels(X, X.clone(), False, 1.0, True, [1.0], "Y = X")[1:]
    print(f"  Y = X: max |dX| {float(gX.abs().max()):.3g}")


@pytest.mark.gpu
def test_lara_layout_per_element(cuda_device):
    """LaRa's layout: V = 8 planar 512^2 views read side by side (scene_loss(ms_ssim=True)'s call, upstream -0.5 of
    loss.backward() with B = 1), bit for bit the ms_ssim_views node; and the channel-last MS_SSIM module's layout on one
    [1,3,512,4096] scene."""
    from lara_b200.ssim import ms_ssim_views
    V, H, W = 8, 512, 512
    img, tar = _inputs(V, 3, H, W, 0, False, 21, 1.0, cuda_device)
    tar = tar.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)       # scene_loss's [V,H,W,3] target
    _, out, gX = check_kernels(img, tar, True, 1.0, True, [-0.5], "LaRa V=8 512^2")
    x = img.clone().requires_grad_(True)
    s = ms_ssim_views(x, tar)
    (0.5 * (1 - s)).backward()
    assert torch.equal(s.reshape(1), out) and torch.equal(x.grad, gX)
    X, Y = _inputs(1, 3, 512, 4096, 0, True, 22, 1.0, cuda_device)
    check_kernels(X, Y, False, 1.0, True, [1.0], "channel-last [1,3,512,4096]")
