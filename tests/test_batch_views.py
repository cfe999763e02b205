"""Host-side checks of the batched scene entries (no GPU needed): the srf_scenes_* argument rejections made before
anything is enqueued, and the shape and settings checks of render_batch_views / render_batch_subset_views."""
import ctypes

import pytest
import torch

from lara_b200 import _lib
from lara_b200 import rasterizer as R
from lara_b200.multiview import batch_view_settings, render_batch_subset_views, render_batch_views


def _fwd_args(S, Vs, tan_fov):
    cams = (ctypes.c_float * 24)()
    return [None, S, Vs, 4, 0, 1, None, None, None, None, None, None, None, ctypes.addressof(cams), tan_fov,
            16, 16, 0, 0, None, None, None, None, None, None, None, None, None, None, 0, 1]


@pytest.mark.parametrize("S,Vs", [(0, 1), (-1, 2), (2, 0), (2, -3), (129, 1), (2, 40000)])
def test_scenes_forward_rejects_bad_counts(lib, S, Vs):
    fov = _lib.tan_fov_array([(1.0, 1.0)] * max(S, 1))
    assert lib.srf_scenes_forward(*_fwd_args(S, Vs, fov)) != 0
    assert b"srf_scenes_forward" in lib.srf_last_error()


@pytest.mark.parametrize("fov", [None, (float("nan"), 1.0), (1.0, float("inf")), (0.0, 1.0), (1.0, -2.0)])
def test_scenes_entries_reject_bad_tan_fov(lib, fov):
    arr = None if fov is None else _lib.tan_fov_array([(1.0, 1.0), fov])
    assert lib.srf_scenes_forward(*_fwd_args(2, 2, arr)) != 0
    assert b"tan_fov" in lib.srf_last_error()
    cams = (ctypes.c_float * 96)()
    bwd = [None, 2, 2, 4, None, 0, 1, 16, 16, 0, ctypes.addressof(cams), None, None, 0, None, None, 0, arr, None,
           None, None, None, None, None, None, None, 0, None, None, None, None, None, None, None, None, 1, 0]
    assert lib.srf_scenes_backward(*bwd) != 0
    assert b"tan_fov" in lib.srf_last_error()


def test_scenes_subset_forward_rejects_bad_sizes(lib):
    def call(S, Vs, P, n, n_max, offsets):
        return lib.srf_scenes_subset_forward(None, S, Vs, P, n, n_max, 0, 1, None, offsets, None, None, None, None, 16,
                                             16, 0, None, None, None, None, 0, 1, None, None, None, None, None, None,
                                             None, None, 1)
    assert call(0, 1, 4, 0, 0, None) != 0 and b"S > 0" in lib.srf_last_error()
    assert call(2, 0, 4, 0, 0, None) != 0
    assert call(2, 1, 4, 0, 5, None) != 0 and b"bad sizes" in lib.srf_last_error()
    assert call(2, 1, 4, 0, 2, None) != 0 and b"null offsets" in lib.srf_last_error()
    assert call(2, 1, 4, 0, 0, None) != 0 and b"null offsets" in lib.srf_last_error()         # NULL offsets with S > 1
    assert call(1, 1, 4, 2, 3, None) != 0 and b"n_max == n" in lib.srf_last_error()        # NULL offsets, n_max != n


def _settings(n, H=16, W=16, fov=1.0, deg=1):
    z = torch.zeros(16)
    return [R.GaussianRasterizationSettings(H, W, fov, fov, torch.zeros(3), 1.0, z, z, deg, torch.zeros(3), False, False)
            for _ in range(n)]


def test_batch_settings_checks():
    H, W, fov, deg, _, _ = batch_view_settings([_settings(2, fov=0.5), _settings(2, fov=0.7)])
    assert (H, W, deg, fov) == (16, 16, 1, [(0.5, 0.5), (0.7, 0.7)])
    with pytest.raises(RuntimeError, match="same number of views"):
        batch_view_settings([_settings(2), _settings(3)])
    with pytest.raises(RuntimeError, match="image size"):
        batch_view_settings([_settings(2), _settings(2, H=32)])
    with pytest.raises(RuntimeError, match="image size and the SH degree"):
        batch_view_settings([_settings(2), _settings(2, deg=2)])
    with pytest.raises(RuntimeError, match="share the field of view"):
        batch_view_settings([_settings(1, fov=0.5) + _settings(1, fov=0.6)])
    with pytest.raises(ValueError):
        batch_view_settings([])


def test_batch_shape_checks():
    B, P = 2, 8
    c, shs, o = torch.zeros(B, P, 3), torch.zeros(B, P, 4, 3), torch.zeros(B, P, 1)
    s, r = torch.zeros(B, P, 2), torch.zeros(B, P, 4)
    st = [_settings(2), _settings(2)]
    with pytest.raises(RuntimeError, match="centers must be"):
        render_batch_views(c[0], shs, o, s, r, st)
    with pytest.raises(RuntimeError, match="shs must be"):
        render_batch_views(c, shs[:, :4], o, s, r, st)
    with pytest.raises(RuntimeError, match="opacity must be"):
        render_batch_views(c, shs, o[:1], s, r, st)
    with pytest.raises(RuntimeError, match="scales"):
        render_batch_views(c, shs, o, s[:, :, :1], r, st)
    with pytest.raises(TypeError):
        render_batch_subset_views(object(), torch.zeros(B, P, dtype=torch.bool), torch.zeros(0, 4, 3))
