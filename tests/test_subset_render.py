"""The subset render's argument checks (``srf_scenes_subset_forward``, ``render_subset_views``), no GPU needed: the C
entry rejects every bad argument before it makes a CUDA call, and the Python entry before it launches anything."""
import ctypes

import pytest
import torch

A = 1 << 20            # a 256-byte aligned address: never dereferenced, the checks fail first
MIS = A + 16


def _args(**kw):
    """srf_scenes_subset_forward's arguments for one scene (S = 1, offsets = NULL) of V = 2 views of a P = 1000 coarse
    forward, n = n_max = 10, 64 x 48, each overridable by name."""
    a = dict(stream=None, S=1, V=2, P=1000, n=10, n_max=None, D=1, M=4, idx=A, offsets=None, means3D=A, shs=A,
             colors_precomp=None, cams=A, H=64, W=48, capacity=4096, coarse_radii=A, coarse_geom=A, coarse_tile=A,
             coarse_point_list=A, coarse_capacity=4096, coarse_for_backward=1, radii=A, geom=A, tile=A, point_list=A,
             image=A, out_color=A, out_others=A, workspace=A, for_backward=1)
    a.update(kw)
    if a["n_max"] is None:
        a["n_max"] = a["n"]
    return list(a.values())


@pytest.mark.parametrize("bad,msg", [
    (dict(n=1001), b"n_max = 1001 > P"),
    (dict(n=-1), b"bad sizes"),
    (dict(V=0), b"Vs > 0"),
    (dict(H=0), b"bad sizes"),
    (dict(D=4), b"sh degree"),
    (dict(M=3), b"SH coefficients"),
    (dict(colors_precomp=A), b"colors_precomp is not supported"),
    (dict(capacity=4095), b"differs from the coarse"),
    (dict(shs=None), b"shs is required"),
    (dict(idx=None), b"null required pointer"),
    (dict(coarse_geom=None), b"null required pointer"),
    (dict(coarse_tile=None), b"null required pointer"),
    (dict(cams=None), b"null required pointer"),
    (dict(image=None), b"null required pointer"),
    (dict(workspace=None), b"null required pointer"),
    (dict(coarse_point_list=None), b"null point list"),
    (dict(workspace=MIS), b"256-byte aligned"),
    (dict(geom=MIS), b"256-byte aligned"),
    (dict(coarse_geom=MIS), b"256-byte aligned"),
    (dict(tile=MIS), b"256-byte aligned"),
    (dict(coarse_point_list=MIS), b"256-byte aligned"),
    (dict(image=MIS), b"256-byte aligned"),
])
def test_scenes_c_entry_rejects_bad_arguments(lib, bad, msg):
    assert lib.srf_scenes_subset_forward(*_args(**bad)) != 0
    err = lib.srf_last_error()
    assert b"srf_scenes_subset_forward" in err and msg in err, err


def test_scenes_c_entry_forward_only_needs_no_image_state(lib):
    # for_backward = 0 takes no image state: the checks then fail only on what is really wrong
    assert lib.srf_scenes_subset_forward(*_args(image=None, for_backward=0, D=5)) != 0
    assert b"sh degree" in lib.srf_last_error()


def test_workspace_query(lib):
    b = ctypes.c_size_t()
    assert lib.srf_views_subset_workspace_bytes(1000, ctypes.byref(b)) == 0
    assert b.value >= 4000 and b.value % 256 == 0
    assert lib.srf_views_subset_workspace_bytes(-1, ctypes.byref(b)) != 0
    assert lib.srf_views_subset_workspace_bytes(0, ctypes.byref(b)) == 0


def _binning(P=50, deg=1):
    """A SceneBinning over CPU tensors: enough for every check render_subset_views makes before a launch."""
    from lara_b200.multiview import SceneBinning
    c, shs, o = torch.zeros(P, 3), torch.zeros(P, (deg + 1) ** 2, 3), torch.zeros(P, 1)
    s, r = torch.zeros(P, 2), torch.zeros(P, 4)
    radii = torch.zeros(2, P, dtype=torch.int32)
    return SceneBinning(None, radii, c, None, (16, 16, 1.0, 1.0, deg, False), None, 0.0, True, (c, shs, o, s, r))


def test_python_checks_raise():
    from lara_b200.multiview import render_subset_views
    b = _binning()
    mask = torch.zeros(50, dtype=torch.bool)
    mask[::3] = True
    shs = torch.zeros(int(mask.sum()), 4, 3)
    with pytest.raises(TypeError):
        render_subset_views({"image": None}, mask, shs)
    for bad in (mask.int(), mask[:-1], mask.view(5, 10), [True] * 50):
        with pytest.raises(RuntimeError, match="mask must be a bool tensor"):
            render_subset_views(b, bad, shs)
    for bad in (shs.double(), shs[:, :3], shs[:, :, :2], shs[0], shs.numpy()):
        with pytest.raises(RuntimeError, match="shs_fine must be float32"):
            render_subset_views(b, mask, bad)
    with pytest.raises(RuntimeError, match="the mask selects"):
        render_subset_views(b, mask, shs[1:])


@pytest.mark.parametrize("which", range(6))
def test_in_place_modification_raises(which):
    from lara_b200.multiview import render_subset_views
    b = _binning()
    (b.tensors + (b.radii,))[which].add_(1)
    mask = torch.ones(50, dtype=torch.bool)
    with pytest.raises(RuntimeError, match="modified in place"):
        render_subset_views(b, mask, torch.zeros(50, 4, 3))


def test_concat_views_skips_the_binning():
    from lara_b200.multiview import concat_views
    out = {"image": torch.zeros(2, 4, 5, 3), "radii": torch.zeros(2, 7), "binning": _binning()}
    assert set(concat_views(out)) == {"image"}
