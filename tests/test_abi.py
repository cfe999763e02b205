"""The C-ABI library loads and exports every symbol include/*.h declares (no GPU needed)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    names = set()
    for fn in os.listdir(os.path.join(ROOT, "include")):
        if fn.endswith(".h"):
            src = open(os.path.join(ROOT, "include", fn)).read()
            src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
            names |= set(re.findall(r"\b(srf_[a-z0-9_]+)\s*\(", src))
    return sorted(names)


def test_header_declares_the_boundary():
    syms = declared_symbols()
    for must in ("srf_forward_preprocess", "srf_forward_render", "srf_backward", "srf_mark_visible",
                 "srf_geom_state_bytes", "srf_last_error"):
        assert must in syms


def test_library_exports_every_declared_symbol(lib):
    for name in declared_symbols():
        assert hasattr(lib, name), f"{name} declared in include/ but not exported"


def test_binding_table_matches_header():
    from lara_b200 import _lib
    assert sorted(_lib.SIGNATURES) == declared_symbols()


def test_abi_version(lib):
    from lara_b200 import _lib
    assert lib.srf_abi_version() == _lib.ABI_VERSION


def test_workspace_sizes_host_only(lib):
    from lara_b200 import _lib
    g, t, i, s = _lib.sizes(lib, 1000, 300, 500)
    assert g >= 1000 * (96 + 4 + 8) and i >= 300 * 500 * 20 and s >= 1000 * 80
    ntiles = ((500 + 15) // 16) * ((300 + 15) // 16)
    assert t >= ntiles * (256 + 8 + 4)
    goff, toff, ioff = _lib.layout(lib, 1000, 300, 500)
    assert goff[0] == 0 and goff[1] >= 96000 and goff[2] >= goff[1] + 4000
    assert all(o % 16 == 0 for o in goff + ioff)
    e, p = _lib.binning_sizes(lib, 12345)
    assert e >= 12345 * 8 and p >= 12345 * 4
    g0, _, _, s0 = _lib.sizes(lib, 0, 16, 16)
    assert g0 > 0 and s0 > 0


def test_bad_arguments_return_status_and_message(lib):
    n = ctypes.c_size_t()
    assert lib.srf_geom_state_bytes(-1, ctypes.byref(n)) != 0
    assert b"srf_geom_state_bytes" in lib.srf_last_error()
    assert lib.srf_tile_state_bytes(0, 16, ctypes.byref(n)) != 0
    # null / misaligned workspaces are rejected before any CUDA call
    args = [None, 4, 0, 1, None, None, None, None, None, 1.0, None, None, None, None, None,
            1.0, 1.0, 16, 16, 0, None, None, None, None, 0]
    assert lib.srf_forward_preprocess(*args) != 0
    assert lib.srf_last_error() != b""


def test_missing_library_fails_loudly(tmp_path):
    from lara_b200 import _lib
    with pytest.raises(_lib.SurfelLibraryError):
        _lib.load(str(tmp_path / "nope.so"))
