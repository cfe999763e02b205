"""Loader + state parser for the reference build in ``oracle/_ref`` (built by
``oracle/build_ref.py`` from a LaRa checkout; git-ignored build output).

TEST INFRASTRUCTURE ONLY: used by ``tests/golden/make_reference_records.py`` (records of the
real reference for the GPU parity tests) and by ``bench.py --impl reference``.  Never imported
by lara_b200/.
"""
from __future__ import annotations

import importlib.util
import os
import sys
from typing import Dict, Optional

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.join(HERE, "_ref", "diff_surfel_rasterization")
MODNAME = "ref_diff_surfel_rasterization"


def available() -> bool:
    return os.path.isfile(os.path.join(PKG, "_C.so")) and os.path.isfile(os.path.join(PKG, "__init__.py"))


def load():
    """Import the unmodified reference package under a distinct module name."""
    if MODNAME in sys.modules:
        return sys.modules[MODNAME]
    if not available():
        raise ImportError("oracle/_ref is not built (LARA_REFERENCE_ROOT=<LaRa checkout> python oracle/build_ref.py)")
    spec = importlib.util.spec_from_file_location(
        MODNAME, os.path.join(PKG, "__init__.py"), submodule_search_locations=[PKG])
    mod = importlib.util.module_from_spec(spec)
    sys.modules[MODNAME] = mod
    spec.loader.exec_module(mod)
    return mod


def _align(x: int, a: int = 128) -> int:
    return (x + a - 1) // a * a


def parse_geom(buf: torch.Tensor, P: int) -> Dict[str, torch.Tensor]:
    """GeometryState::fromChunk (rasterizer_impl.cu:155-170): sub-arrays start on 128 B
    boundaries of the absolute address; torch allocations are >= 512 B aligned."""
    base = buf.data_ptr()
    off = 0
    out = {}

    def take(name, nbytes, dtype, shape):
        nonlocal off
        start = _align(base + off) - base
        out[name] = buf[start:start + nbytes].view(dtype).view(*shape) if nbytes else torch.empty(shape, dtype=dtype)
        off = start + nbytes

    take("depths", 4 * P, torch.float32, (P,))
    take("clamped", 3 * P, torch.uint8, (P, 3))
    take("internal_radii", 4 * P, torch.int32, (P,))
    take("means2D", 8 * P, torch.float32, (P, 2))
    take("transMat", 36 * P, torch.float32, (P, 9))
    take("normal_opacity", 16 * P, torch.float32, (P, 4))
    take("rgb", 12 * P, torch.float32, (P, 3))
    take("tiles_touched", 4 * P, torch.int32, (P,))
    return out


def parse_image(buf: torch.Tensor, H: int, W: int, ntiles: int) -> Dict[str, torch.Tensor]:
    """ImageState::fromChunk (rasterizer_impl.cu:172-179)."""
    N = H * W
    base = buf.data_ptr()
    o0 = _align(base) - base
    accum = buf[o0:o0 + 12 * N].view(torch.float32).view(3, H, W)
    o1 = _align(base + o0 + 12 * N) - base
    n_contrib = buf[o1:o1 + 8 * N].view(torch.int32).view(2, H, W)
    o2 = _align(base + o1 + 8 * N) - base
    ranges = buf[o2:o2 + 8 * ntiles].view(torch.int32).view(ntiles, 2)
    return {"accum": accum, "n_contrib": n_contrib, "ranges": ranges}


def parse_binning(buf: torch.Tensor, R: int) -> Dict[str, torch.Tensor]:
    """BinningState::fromChunk (rasterizer_impl.cu:181-194): point_list is first."""
    base = buf.data_ptr()
    o0 = _align(base) - base
    return {"point_list": buf[o0:o0 + 4 * R].view(torch.int32)}


def forward_raw(ref, sc: Dict[str, torch.Tensor], settings) -> Dict[str, object]:
    """Call the reference's native forward directly (to get at its state blobs)."""
    dev = sc["means3D"].device
    empty = torch.empty(0, device=dev)
    shs = sc.get("shs")
    colors = sc.get("colors_precomp")
    args = (settings.bg, sc["means3D"], colors if colors is not None else empty, sc["opacities"],
            sc["scales"], sc["rotations"], settings.scale_modifier, empty, settings.viewmatrix,
            settings.projmatrix, settings.tanfovx, settings.tanfovy, settings.image_height,
            settings.image_width, shs if shs is not None else empty, settings.sh_degree, settings.campos,
            settings.prefiltered, settings.debug)
    R, color, allmap, radii, geom, binning, img = ref._C.rasterize_gaussians(*args)
    P = sc["means3D"].shape[0]
    H, W = settings.image_height, settings.image_width
    ntiles = ((W + 15) // 16) * ((H + 15) // 16)
    out = {"num_rendered": int(R), "color": color, "allmap": allmap, "radii": radii,
           "geomBuffer": geom, "binningBuffer": binning, "imgBuffer": img}
    if P > 0:
        out.update(parse_geom(geom, P))
        out.update(parse_image(img, H, W, ntiles))
        out.update(parse_binning(binning, int(R)))
    return out
