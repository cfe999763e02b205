"""LaRa's evaluation on the GPU (lara_b200.ssim.ssim, lara_b200.evaluate), CPU side.

* The single-scale SSIM contract (pytorch-msssim 1.0.0 ``ssim``): a plain-torch restatement built on test_ms_ssim's
  ``_ssim`` equals an independent float64 NumPy/SciPy statement with a hand-written vjp.
* ``video_path``'s cameras and the frame rounding chain equal what LaRa's own ``tools/gen_video_path.py`` and
  ``evaluation.py:132-136`` lines compute on the CPU, recorded in tests/golden/reference/test_eval.npz
  (``record_reference``; ``python tests/test_eval.py OUT_DIR LARA_CHECKOUT`` writes OUT_DIR/test_eval.npz with
  tests/golden/make_reference_records.py's writer).
* The new C entries reject bad arguments before any launch.
"""
from __future__ import annotations

import ctypes
import importlib
import os
import sys
import types

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from helpers import reference_record  # noqa: E402
from test_ms_ssim import _fspecial_gauss_1d, _ssim, np_window, smooth_pair  # noqa: E402


# ---- SSIM: plain-torch restatement and a float64 NumPy statement ----

def ssim_torch(X, Y, data_range=255, size_average=True, nonnegative_ssim=False):
    """pytorch-msssim 1.0.0 ``ssim`` for 4-D inputs with the default window and K, in the library's torch calls."""
    win = _fspecial_gauss_1d(11, 1.5).repeat([X.shape[1], 1, 1, 1])
    ssim_per_channel, _ = _ssim(X, Y, data_range=data_range, win=win)
    if nonnegative_ssim:
        ssim_per_channel = torch.relu(ssim_per_channel)
    return ssim_per_channel.mean() if size_average else ssim_per_channel.mean(1)


def np_ssim(X, Y, data_range=255, size_average=True, nonnegative_ssim=False):
    """(value, d sum(value) / dX) in float64: a valid 2-D correlation with the outer-product window and the vjp
    written out: dX = (G^T A + 2 X G^T B + Y G^T C) / count per plane, A = dS/dmu_x, B = dS/dG(XX), C = dS/dG(XY)."""
    from scipy.signal import convolve2d, correlate2d
    g1 = _fspecial_gauss_1d(11, 1.5).reshape(-1).numpy().astype(np.float64)    # the window at its own fp32 precision
    assert np.abs(np_window() - g1).max() <= 2 * np.finfo(np.float32).eps * g1.max()
    k2 = np.outer(g1, g1)
    C1, C2 = (0.01 * data_range) ** 2, (0.03 * data_range) ** 2
    B, C = X.shape[:2]
    vals, grads = np.zeros((B, C)), np.zeros(X.shape)
    for b in range(B):
        for c in range(C):
            x, y = X[b, c], Y[b, c]
            f = lambda a: correlate2d(a, k2, mode="valid")      # noqa: E731
            mx, my, gxx, gyy, gxy = f(x), f(y), f(x * x), f(y * y), f(x * y)
            sx, sy, sxy = gxx - mx * mx, gyy - my * my, gxy - mx * my
            D, Dl = sx + sy + C2, mx * mx + my * my + C1
            cs, lum = (2 * sxy + C2) / D, (2 * mx * my + C1) / Dl
            m = (lum * cs).mean()
            keep = not nonnegative_ssim or m > 0
            vals[b, c] = m if keep else 0.0
            A = cs * 2 * (my - mx * lum) / Dl + lum * 2 * (mx * cs - my) / D
            Bm, Cm = lum * -cs / D, lum * 2 / D
            g = lambda a: convolve2d(a, k2, mode="full")        # noqa: E731
            grads[b, c] = (g(A) + 2 * x * g(Bm) + y * g(Cm)) / cs.size if keep else 0.0
    scale = 1.0 / (B * C if size_average else C)
    return (vals.mean() if size_average else vals.mean(1)), grads * scale


SSIM_CASES = {
    # name: (B, C, H, W, seed, data_range, size_average, nonnegative_ssim, negative plane)
    "odd_23x37": (2, 3, 23, 37, 1, 1.0, True, False, False),
    "per_batch_19x11": (3, 3, 19, 11, 2, 1.0, False, False, False),
    "range255_11x29": (1, 3, 11, 29, 3, 255.0, True, False, False),
    "nonnegative_with_negative_plane": (2, 3, 31, 27, 4, 1.0, False, True, True),
    "signed_negative_plane": (2, 3, 31, 27, 4, 1.0, True, False, True),
}


def ssim_pair(B, C, H, W, seed, negative):
    X, Y = smooth_pair(B, C, H, W, seed)
    if negative:        # plane (0, 1): anti-correlated target, a negative mean ssim
        Y[0, 1] = 2 * X[0, 1].mean() - X[0, 1]
    return X, Y


@pytest.mark.parametrize("case", list(SSIM_CASES))
def test_ssim_restatement_matches_numpy_statement_float64(case):
    B, C, H, W, seed, R, size_average, nonneg, negative = SSIM_CASES[case]
    X, Y = ssim_pair(B, C, H, W, seed, negative)
    X, Y = X * R, Y * R
    Xg = X.clone().requires_grad_(True)
    v = ssim_torch(Xg, Y, R, size_average, nonneg)
    v.sum().backward()
    v_np, g_np = np_ssim(X.numpy(), Y.numpy(), R, size_average, nonneg)
    if negative:
        per_channel, _ = _ssim(X, Y, R, _fspecial_gauss_1d(11, 1.5).repeat([C, 1, 1, 1]))
        assert float(per_channel[0, 1]) < 0
    assert np.abs(v.detach().numpy() - v_np).max() <= 1e-12 * np.abs(v_np).max()
    assert np.abs(Xg.grad.numpy() - g_np).max() <= 1e-12 * np.abs(g_np).max()
    if nonneg and negative:
        assert float(np.abs(Xg.grad[0, 1]).max()) == 0.0


def test_ssim_argument_checks():
    from lara_b200.ssim import SSIM, ssim, ssim_views
    X = torch.zeros(1, 3, 16, 16)
    with pytest.raises(ValueError, match="win_size"):
        ssim(X, X, win_size=7)
    with pytest.raises(ValueError, match="K"):
        SSIM(K=(0.02, 0.03))
    with pytest.raises(ValueError, match="at least the window size 11"):
        ssim(torch.zeros(1, 3, 10, 16), torch.zeros(1, 3, 10, 16))
    with pytest.raises(TypeError, match="float32"):
        ssim(X.double(), X.double())
    with pytest.raises(ValueError, match="view range"):
        ssim_views(torch.zeros(4, 3, 16, 16), torch.zeros(4, 3, 16, 16), view_range=(4, 4))


# ---- LaRa's video path and frame expressions, recorded ----

def _import_lara_video_path(lara):
    """LaRa's tools/gen_video_path.py with stubs for what its imports pull in but the path never uses."""
    stubs = {}

    def stub(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        stubs[name] = m
        return m

    class _Any:
        def __class_getitem__(cls, item):
            return cls
    stub("sklearn").cluster = stub("sklearn.cluster", KMeans=object)
    stub("jaxtyping", Float=_Any)
    saved = {k: sys.modules.get(k) for k in stubs}
    mods = ("tools", "dataLoader")
    sys.modules.update(stubs)
    sys.path.insert(0, lara)
    try:
        for k in [k for k in sys.modules if k.split(".")[0] in mods]:
            del sys.modules[k]
        utils = importlib.util.spec_from_file_location("dataLoader.utils", os.path.join(lara, "dataLoader", "utils.py"))
        du = importlib.util.module_from_spec(utils)
        sys.modules["dataLoader"] = types.ModuleType("dataLoader")
        sys.modules["dataLoader.utils"] = du
        utils.loader.exec_module(du)
        return importlib.import_module("tools.gen_video_path")
    finally:
        sys.path.remove(lara)
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


class _Cfg:
    def __init__(self, name, img_size):
        self.dataset_name, self.img_size = name, list(img_size)


def _transform(seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.nn.functional.normalize(torch.randn(4, generator=g, dtype=torch.float64), dim=0)
    w, x, y, z = q.tolist()
    m = torch.eye(4)
    m[:3, :3] = torch.tensor([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                              [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                              [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    return m[None, None]        # sample['transform_mats'] is [B, 1, 4, 4]


PATH_CASES = {
    # name: (dataset, N, img_size (w, h), transform seed or None, fov or None, elevation)
    "gobjeverse_120": ("gobjeverse", 120, (512, 512), None, (0.9, 0.8), 0),
    "GSO_sample_elev30": ("GSO", 7, (64, 48), 5, None, 30),
    "instant3d_fov": ("instant3d", 9, (512, 512), None, (0.6, 0.5), 0),
    "mvgen_sample_elev-30": ("mvgen", 5, (40, 56), 6, None, -30),
}
CAM_FIELDS = ("world_view_transform", "full_proj_transform", "camera_center")


def _frame_inputs(seed=7, N=2, H=37, W=41):
    """fp32 renders that include every exact half (k + 0.5) / 255, 0, 1 and the saturating ends."""
    g = torch.Generator().manual_seed(seed)
    img = torch.rand((N, H, W, 3), generator=g)
    k = torch.arange(256, dtype=torch.float32)
    flat = img.view(-1)
    flat[:256] = (k + 0.5) / 255
    flat[256:512] = k / 255
    flat[512:520] = torch.tensor([0.0, 1.0, -0.01, 1.01, 0.5 / 255, 254.5 / 255, 1e-8, 0.999999])
    normal = torch.rand((N, H, W, 3), generator=g) * 2 - 1
    alpha = torch.rand((N, H, W), generator=g)
    alpha.view(-1)[:64] = torch.tensor([0.0, 1.0] * 32)
    return img, normal, alpha


def lara_frames(img, normal, alpha):
    """evaluation.py:132-136 on the CPU, line for line."""
    rgb = np.round(img.numpy() * 255).astype("uint8")
    a = alpha[..., None]
    nrm = np.round((((normal * a + 1 - a) + 1) / 2).numpy() * 255).astype("uint8")
    return rgb, nrm


def record_reference(lara, dev):
    """LaRa's camera path and frame expressions on the CPU, run by this file's ``__main__``."""
    gvp = _import_lara_video_path(lara)
    recs = {}
    for case, (name, N, size, seed, fov, elev) in PATH_CASES.items():
        sample = None if seed is None else {"transform_mats": _transform(seed)}
        fovt = None if fov is None else [torch.tensor([fov[0]]), torch.tensor([fov[1]])]
        gen = gvp.generate_gobjverse_frames if name in ("gobjeverse", "GSO") else gvp.generate_instant3d_frames
        cams = gen(N, _Cfg(name, size), sample, elevation=elev, fov=fovt)
        r = {f: np.stack([getattr(c, f).numpy() for c in cams]) for f in CAM_FIELDS}
        r["fov"] = np.array([[c.FoVx, c.FoVy] for c in cams])
        r["size"] = np.array([[c.image_width, c.image_height] for c in cams])
        if elev == 0:     # uni_video_path passes no elevation
            assert all(np.array_equal(a.world_view_transform.numpy(), b.world_view_transform.numpy())
                       for a, b in zip(cams, gvp.uni_video_path(N, _Cfg(name, size), sample, fov=fovt)))
        recs[case] = r
    img, normal, alpha = _frame_inputs()
    rgb, nrm = lara_frames(img, normal, alpha)
    recs["frames"] = {"rgb": rgb, "nrm": nrm}
    return recs


def _path(case):
    from lara_b200.evaluate import video_path
    name, N, size, seed, fov, elev = PATH_CASES[case]
    sample = None if seed is None else {"transform_mats": _transform(seed)}
    fovt = None if fov is None else [torch.tensor([fov[0]]), torch.tensor([fov[1]])]
    return video_path(N, name, size, sample=sample, fov=fovt, elevation=elev)


@pytest.mark.parametrize("case", list(PATH_CASES))
def test_video_path_equals_lara_record(case):
    rec = reference_record("test_eval", case)
    cams = _path(case)
    for f in CAM_FIELDS:
        mine = np.stack([getattr(c, f).numpy() for c in cams])
        assert mine.dtype == rec[f].dtype and np.array_equal(mine, rec[f]), f
    assert np.array_equal(np.array([[c.FoVx, c.FoVy] for c in cams]), rec["fov"])
    assert np.array_equal(np.array([[c.image_width, c.image_height] for c in cams]), rec["size"])


def test_video_path_unposed_is_not_restated():
    from lara_b200.evaluate import video_path
    with pytest.raises(NotImplementedError):
        video_path(4, "unposed", (64, 64))


def frames_chain_np(img, normal, alpha):
    """srf_video_frames' chain in NumPy fp32, each operation rounded on its own, np.rint half to even, saturation."""
    f = np.float32
    q = lambda v: np.clip(np.rint(v), 0, 255).astype(np.uint8)      # noqa: E731
    a = alpha[..., None].astype(f)
    t = ((((normal.astype(f) * a).astype(f) + f(1)).astype(f) - a).astype(f) + f(1)).astype(f) * f(0.5)
    return q(img.astype(f) * f(255)), q(t.astype(f) * f(255))


def test_frame_chain_equals_lara_record():
    rec = reference_record("test_eval", "frames")
    img, normal, alpha = _frame_inputs()
    rgb, nrm = frames_chain_np(img.numpy(), normal.numpy(), alpha.numpy())
    inside = (img.numpy() >= 0) & (img.numpy() <= 1)
    assert np.array_equal(rgb[inside], rec["rgb"][inside])
    assert np.array_equal(nrm, rec["nrm"])
    # the halves round to even, as np.round does
    assert list(rec["rgb"].reshape(-1)[:4]) == [0, 2, 2, 4]


# ---- C entries: argument checks before any launch ----

def test_c_entries_reject_bad_arguments_before_any_launch(lib):
    from lara_b200 import _lib
    n = ctypes.c_size_t()
    assert lib.srf_ssim_workspace_bytes(1, 3, 10, 64, ctypes.byref(n)) != 0
    assert b"at least the window size 11" in lib.srf_last_error()
    assert lib.srf_ssim_workspace_bytes(1, 3, 11, 11, ctypes.byref(n)) == 0 and n.value % 256 == 0
    assert lib.srf_ssim_workspace_bytes(300, 300, 11, 11, ctypes.byref(n)) != 0
    a = _lib.MsSsimAddr(0, 121, 11, 1, 0, 11)
    fwd = lambda ws, B=1, H=11, out=4096: lib.srf_ssim_forward(None, B, 3, H, 11, 256, ctypes.byref(a), 512,  # noqa
                                                                 ctypes.byref(a), 1.0, 1, 0, ws, out)
    assert fwd(None) != 0 and b"workspace" in lib.srf_last_error()
    assert fwd(1024 + 16) != 0 and b"workspace" in lib.srf_last_error()
    assert fwd(1024, B=0) != 0 and b"bad sizes" in lib.srf_last_error()
    assert fwd(1024, H=7) != 0
    assert fwd(1024, out=None) != 0 and b"output" in lib.srf_last_error()
    assert lib.srf_ssim_backward(None, 1, 3, 11, 11, 256, ctypes.byref(a), 512, ctypes.byref(a), 1.0, 1, 0, 1024,
                                 None, 2048, ctypes.byref(a)) != 0
    assert b"upstream" in lib.srf_last_error()

    assert lib.srf_eval_workspace_bytes(ctypes.byref(n)) == 0 and n.value > 0
    thr = (ctypes.c_double * 9)(*([0.1] * 9))

    def metrics(V=2, v0=1, v1=2, ws=1024, out=2048, nthr=0, depth=None, image=256):
        return lib.srf_eval_metrics(None, V, 16, 16, v0, v1, image, ctypes.byref(a), 512, ctypes.byref(a), depth,
                                    ctypes.byref(a), 768, ctypes.byref(a), 4096, ctypes.byref(a), nthr, thr, ws, out)
    assert metrics(v0=2, v1=1) != 0 and b"view range" in lib.srf_last_error()
    assert metrics(v1=3) != 0 and b"view range" in lib.srf_last_error()
    assert metrics(V=0) != 0 and b"bad sizes" in lib.srf_last_error()
    assert metrics(nthr=9) != 0 and b"n_thresholds" in lib.srf_last_error()
    assert metrics(ws=None) != 0 and b"workspace" in lib.srf_last_error()
    assert metrics(ws=1024 + 8) != 0 and b"workspace" in lib.srf_last_error()
    assert metrics(out=2052) != 0 and b"out" in lib.srf_last_error()
    assert metrics(image=None) != 0 and b"image" in lib.srf_last_error()
    assert metrics(image=258) != 0 and b"aligned" in lib.srf_last_error()
    assert metrics(depth=1026) != 0 and b"depth" in lib.srf_last_error()

    def frames(N=2, image=256, rgb=4096, normal=None, alpha=None, nrm=None):
        return lib.srf_video_frames(None, N, 16, 16, image, ctypes.byref(a), normal, ctypes.byref(a), alpha,
                                    ctypes.byref(a), rgb, nrm)
    assert frames(N=-1) != 0 and b"bad sizes" in lib.srf_last_error()
    assert frames(rgb=None) != 0 and b"rgb" in lib.srf_last_error()
    assert frames(normal=512, alpha=None, nrm=8192) != 0 and b"alpha" in lib.srf_last_error()
    assert frames(normal=512, alpha=768, nrm=None) != 0 and b"nrm" in lib.srf_last_error()
    assert frames(image=254) != 0 and b"aligned" in lib.srf_last_error()


if __name__ == "__main__":
    # python tests/test_eval.py OUT_DIR LARA_CHECKOUT, then cp OUT_DIR/test_eval.npz tests/golden/reference/
    spec = importlib.util.spec_from_file_location(
        "make_reference_records", os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                                               "make_reference_records.py"))
    writer = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(writer)
    os.makedirs(sys.argv[1], exist_ok=True)
    writer.save(sys.argv[1], "test_eval", record_reference(sys.argv[2], "cpu"))
