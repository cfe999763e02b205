"""ctypes binding of ``libsurfel_b200.so`` (the C ABI in include/surfel_rasterizer.h).

There is no fallback path: if the shared library is missing or does not export
the expected ABI the import of :mod:`lara_b200` still succeeds (so that LaRa's
CPU-only plumbing can import ``diff_surfel_rasterization``), but the first use of
the rasterizer raises ``RuntimeError`` loudly.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int, c_size_t, c_void_p

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libsurfel_b200.so")
ABI_VERSION = 6
CAM_FLOATS, CAM_VIEW, CAM_CAMPOS, CAM_BG = 24, 0, 16, 19      # include/surfel_rasterizer.h SRF_CAM_*

# name -> (restype, argtypes); mirrors include/surfel_rasterizer.h one to one
_P = c_void_p
SIGNATURES = {
    "srf_abi_version": (c_int, []),
    "srf_last_error": (c_char_p, []),
    "srf_geom_state_bytes": (c_int, [c_int, POINTER(c_size_t)]),
    "srf_tile_state_bytes": (c_int, [c_int, c_int, POINTER(c_size_t)]),
    "srf_image_state_bytes": (c_int, [c_int, c_int, POINTER(c_size_t)]),
    "srf_binning_bytes": (c_int, [c_size_t, POINTER(c_size_t), POINTER(c_size_t)]),
    "srf_backward_scratch_bytes": (c_int, [c_int, POINTER(c_size_t)]),
    "srf_state_layout": (c_int, [c_int, c_int, c_int, POINTER(c_size_t), POINTER(c_size_t), POINTER(c_size_t)]),
    "srf_forward_preprocess": (c_int, [
        _P, c_int, c_int, c_int,            # stream, P, D, M
        _P, _P, _P,                         # means3D, shs, colors_precomp
        _P, _P, c_float,                    # opacities, scales, scale_modifier
        _P, _P,                             # rotations, transMat_precomp
        _P, _P, _P,                         # viewmatrix, projmatrix, campos
        c_float, c_float, c_int, c_int,     # tan_fovx, tan_fovy, H, W
        c_int,                              # prefiltered
        _P, _P, _P,                         # radii, geom_state, tile_state
        _P,                                 # num_rendered_host
        c_int,                              # raw_activations
    ]),
    "srf_forward_render": (c_int, [
        _P, c_int, c_int, c_int,            # stream, P, H, W
        c_size_t, _P, _P,                   # capacity, geom_state, tile_state
        _P, _P, _P,                         # entries, point_list, image_state
        _P, _P, _P,                         # background, out_color, out_others
    ]),
    "srf_forward": (c_int, [
        _P, c_int, c_int, c_int,            # stream, P, D, M
        _P, _P, _P,                         # means3D, shs, colors_precomp
        _P, _P, c_float,                    # opacities, scales, scale_modifier
        _P, _P,                             # rotations, transMat_precomp
        _P, _P, _P,                         # viewmatrix, projmatrix, campos
        c_float, c_float, c_int, c_int,     # tan_fovx, tan_fovy, H, W
        c_int,                              # prefiltered
        _P, c_size_t,                       # background, capacity
        _P, _P, _P, _P, _P, _P,             # radii, geom_state, tile_state, entries, point_list, image_state
        _P, _P, _P, _P,                     # out_color, out_others, num_rendered_host, count_event
        c_int,                              # raw_activations
    ]),
    "srf_backward": (c_int, [
        _P, c_int, c_int, c_int, c_int, c_int,   # stream, P, D, M, H, W
        c_size_t, _P,                            # capacity, background
        _P, _P, c_int,                           # means3D, shs, colors_were_precomputed
        _P, _P, c_int,                           # scales, rotations, transmat_was_precomputed
        _P, _P, _P,                              # viewmatrix, projmatrix, campos
        c_float, c_float, _P,                    # tan_fovx, tan_fovy, radii
        _P, _P, _P, _P,                          # geom_state, tile_state, point_list, image_state
        _P, _P,                                  # dL_dout_color, dL_dout_others
        _P, c_int,                               # scratch, accumulate
        _P, _P, _P, _P,                          # dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors
        _P, _P, _P, _P,                          # dL_dopacity, dL_dscales, dL_drotations, dL_dtransMat
        c_int,                                   # raw_activations
    ]),
    "srf_views_workspace_bytes": (c_int, [c_int, c_int, c_int, c_int, c_size_t, POINTER(c_size_t)]),
    "srf_views_forward_preprocess": (c_int, [
        _P, c_int, c_int, c_int, c_int,     # stream, V, P, D, M
        _P, _P, _P,                         # means3D, shs, colors_precomp
        _P, _P, _P,                         # opacities, scales, rotations
        _P, _P,                             # transMat_precomp, cams
        c_float, c_float, c_int, c_int,     # tan_fovx, tan_fovy, H, W
        c_int,                              # prefiltered
        _P, _P, _P,                         # radii, geom_state, tile_state
        _P,                                 # num_rendered_host
        c_int,                              # raw_activations
    ]),
    "srf_views_forward_render": (c_int, [
        _P, c_int, c_int, c_int, c_int,     # stream, V, P, H, W
        c_size_t, _P, _P,                   # capacity, geom_state, tile_state
        _P, _P, _P,                         # entries, point_list, image_state
        _P, _P, _P,                         # cams, out_color, out_others
    ]),
    "srf_views_backward": (c_int, [
        _P, c_int, c_int, c_int, c_int, c_int, c_int,   # stream, V, P, D, M, H, W
        c_size_t, _P,                            # capacity, cams
        _P, _P, c_int,                           # means3D, shs, colors_were_precomputed
        _P, _P, c_int,                           # scales, rotations, transmat_was_precomputed
        c_float, c_float, _P,                    # tan_fovx, tan_fovy, radii
        _P, _P, _P, _P,                          # geom_state, tile_state, point_list, image_state
        _P, _P,                                  # dL_dout_color, dL_dout_others
        _P, c_int,                               # scratch, accumulate
        _P, _P, _P, _P,                          # dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors
        _P, _P, _P, _P,                          # dL_dopacity, dL_dscales, dL_drotations, dL_dtransMat
        c_int,                                   # raw_activations
    ]),
    "srf_views_epilogue_forward": (c_int, [_P, c_int, c_int, c_int, c_float, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "srf_views_epilogue_backward": (c_int, [_P, c_int, c_int, c_int, c_float, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "srf_loss_forward": (c_int, [_P, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, _P, _P]),
    "srf_loss_backward": (c_int, [_P, c_int, c_int, c_int, c_int, c_float, c_float, c_float, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "srf_decoder_layout_forward": (c_int, [_P, c_size_t, c_int, c_int, c_int, c_float, c_float, c_float, _P, _P, _P, _P, _P, _P, _P]),
    "srf_decoder_layout_backward": (c_int, [_P, c_size_t, c_int, c_int, c_int, c_float, _P, _P, _P, _P, _P, _P, _P]),
    "srf_point_feats_forward": (c_int, [_P, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, _P, _P, _P]),
    "srf_point_feats_backward": (c_int, [_P, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "srf_mark_visible": (c_int, [_P, c_int, _P, _P, _P, _P]),
    "srf_epilogue_forward": (c_int, [_P, c_int, c_int, c_float, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "srf_epilogue_backward": (c_int, [_P, c_int, c_int, c_float, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "srf_profile_begin": (c_int, []),
    "srf_profile_end": (c_int, [POINTER(c_float), POINTER(c_int), c_int]),
}

_lib = None


class SurfelLibraryError(RuntimeError):
    pass


def load(path: str | None = None):
    """Load (once) and return the ctypes handle; raises if the library is unusable."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.isfile(p):
        raise SurfelLibraryError(
            f"{p} not found: the CUDA extension is not built. Run `python -m lara_b200.build` "
            "(or __graft_entry__.build()). There is no CPU or PyTorch fallback for the rasterizer.")
    lib = ctypes.CDLL(p)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as ex:
            raise SurfelLibraryError(f"{p} does not export {name}; rebuild the extension") from ex
        fn.restype = res
        fn.argtypes = args
    if lib.srf_abi_version() != ABI_VERSION:
        raise SurfelLibraryError(f"{p}: ABI version {lib.srf_abi_version()} != expected {ABI_VERSION}")
    if path is None:
        _lib = lib
    return lib


def check(status: int, lib=None) -> None:
    if status != 0:
        l = lib or _lib
        msg = l.srf_last_error().decode("utf-8", "replace") if l is not None else "unknown error"
        raise RuntimeError(msg)


def sizes(lib, P: int, H: int, W: int):
    g, t, i, s = c_size_t(), c_size_t(), c_size_t(), c_size_t()
    check(lib.srf_geom_state_bytes(P, ctypes.byref(g)), lib)
    check(lib.srf_tile_state_bytes(H, W, ctypes.byref(t)), lib)
    check(lib.srf_image_state_bytes(H, W, ctypes.byref(i)), lib)
    check(lib.srf_backward_scratch_bytes(P, ctypes.byref(s)), lib)
    return g.value, t.value, i.value, s.value


def binning_sizes(lib, capacity: int):
    e, p = c_size_t(), c_size_t()
    check(lib.srf_binning_bytes(capacity, ctypes.byref(e), ctypes.byref(p)), lib)
    return e.value, p.value


def views_sizes(lib, V: int, P: int, H: int, W: int, capacity: int):
    """(geom, tile, image, entries, point_list, backward scratch) bytes for V back-to-back per-view workspaces."""
    b = (c_size_t * 6)()
    check(lib.srf_views_workspace_bytes(V, P, H, W, capacity, b), lib)
    return tuple(int(x) for x in b)


def layout(lib, P: int, H: int, W: int):
    g = (c_size_t * 3)()
    t = (c_size_t * 5)()
    i = (c_size_t * 2)()
    check(lib.srf_state_layout(P, H, W, g, t, i), lib)
    return list(g), list(t), list(i)


KERNEL_NAMES = ["preprocess_fwd", "tile_scan", "scatter", "sort_small", "sort_big", "render_fwd",
                "render_bwd", "preprocess_bwd"]


def profile_begin(lib=None) -> None:
    l = lib or load()
    check(l.srf_profile_begin(), l)


def profile_end(lib=None):
    """Returns {kernel name: (total ms, launches)} for the launches since profile_begin()."""
    l = lib or load()
    n = len(KERNEL_NAMES)
    ms = (c_float * n)()
    cnt = (c_int * n)()
    check(l.srf_profile_end(ms, cnt, n), l)
    return {KERNEL_NAMES[i]: (float(ms[i]), int(cnt[i])) for i in range(n)}
