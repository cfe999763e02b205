"""The blend forward's per-tile cull (surfel_common.cuh: octagon_block_bits) against the per-block test it stands for.

The thread that stages a splat tests its conservative octagon against all eight 8x4 blocks of the tile at once and keeps
one byte; warp b of the tile then keeps the splats with bit b set.  Every hit list, pixel mask and output of the blend
stays the same only if bit b equals octagon_hits(q2, q5, make_warp_rect(tile_x, tile_y, b)) exactly.  A host build of
the header compares the two for every (splat, tile) pair of:

* the bench scene's splats (131 072 Gaussians, a 512 x 512 view), at tiles in the image centre and on its border;
* the far-from-origin and faint-splat windows of test_cull_invariant.py (1024 x 1024);
* unbounded octagons (the tau-ellipse crosses the camera plane: fp16 infinities), empty ones (opacity < 1/255), and
  octagons whose edges fall exactly on the blocks' pixel-centre bounds.

The octagons come from the numpy restatement of preprocess.cu in test_cull_invariant.py; the centres and homographies
from the CPU oracle."""
import os
import subprocess

import numpy as np
import pytest
import torch

from lara_b200 import scene as S
from oracle import oracle as O
from test_cull_invariant import _octagon

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "lara_b200", "csrc")
f32 = np.float32

_SRC = r"""
#include "surfel_common.cuh"
#include <stdio.h>
#include <stdlib.h>

// argv: records file (n x [q2, q5] as 8 floats), tiles file (m x [tile_x, tile_y] as int32), output file (n x m x 2 bytes:
// octagon_block_bits, then the eight octagon_hits results packed the same way)
int main(int argc, char** argv) {
    FILE* fr = fopen(argv[1], "rb"); FILE* ft = fopen(argv[2], "rb");
    fseek(fr, 0, SEEK_END); const long n = ftell(fr) / 32; fseek(fr, 0, SEEK_SET);
    fseek(ft, 0, SEEK_END); const long m = ftell(ft) / 8; fseek(ft, 0, SEEK_SET);
    float4* rec = (float4*)malloc(n * 32); int* tiles = (int*)malloc(m * 8);
    if (fread(rec, 32, n, fr) != (size_t)n || fread(tiles, 8, m, ft) != (size_t)m) return 2;
    unsigned char* out = (unsigned char*)malloc(n * m * 2);
    for (long i = 0; i < n; ++i)
        for (long t = 0; t < m; ++t) {
            const float4 q2 = rec[2 * i], q5 = rec[2 * i + 1];
            const int tx = tiles[2 * t], ty = tiles[2 * t + 1];
            unsigned ref = 0;
            for (int b = 0; b < 8; ++b) ref |= (unsigned)octagon_hits(q2, q5, make_warp_rect(tx, ty, b)) << b;
            out[2 * (i * m + t)] = (unsigned char)octagon_block_bits(q2, q5, tx, ty);
            out[2 * (i * m + t) + 1] = (unsigned char)ref;
        }
    FILE* fo = fopen(argv[3], "wb");
    fwrite(out, 1, n * m * 2, fo);
    fclose(fo);
    printf("pairs %ld\n", n * m);
    return 0;
}
"""


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    from lara_b200 import build
    d = tmp_path_factory.mktemp("block_cull")
    src = d / "block_cull.cu"
    src.write_text(_SRC)
    exe = str(d / "block_cull")
    subprocess.run([build._nvcc(), "-O2", "-std=c++17", "-I", CSRC, "-Xcompiler", "-ffp-contract=off",
                    "-gencode", "arch=compute_90a,code=sm_90a", str(src), "-o", exe], check=True, timeout=600)
    return d, exe


def _records(centre, tw_z, opac, lo, hi):
    """[n, 8] float32: q2 = (Tw.z, cx, cy, opacity), q5 = the eight fp16 offsets as preprocess.cu packs them."""
    n = centre.shape[0]
    q2 = np.stack([tw_z, centre[:, 0], centre[:, 1], opac], axis=1).astype(f32)
    halves = np.stack([lo, hi], axis=2).astype(np.float16).reshape(n, 8)   # (lo, hi) per axis: low half first
    q5 = halves.view(np.uint32).view(f32).reshape(n, 4)
    return np.ascontiguousarray(np.concatenate([q2, q5], axis=1))


def _compare(checker, rec, tiles):
    d, exe = checker
    rec_path, tile_path, out_path = d / "rec.bin", d / "tiles.bin", d / "out.bin"
    rec.astype(f32).tofile(rec_path)
    np.asarray(tiles, dtype=np.int32).reshape(-1, 2).tofile(tile_path)
    subprocess.run([exe, str(rec_path), str(tile_path), str(out_path)], check=True, capture_output=True, timeout=600)
    out = np.fromfile(out_path, dtype=np.uint8).reshape(rec.shape[0], len(tiles), 2)
    bits, ref = out[..., 0], out[..., 1]
    bad = int((bits != ref).sum())
    assert bad == 0, f"{bad} of {bits.size} (splat, tile) bytes differ from the eight per-block tests"
    return bits


def _scene_records(P, size, seed, opacities=None, scale=1.0):
    sc = S.scene(P, seed)
    if opacities is not None:
        sc["opacities"] = opacities
    sc["scales"] = sc["scales"] * scale
    cam = S.cameras(3, size, size, seed)[seed % 3]
    O.load()
    run = O.run_scene(sc, cam, torch.ones(3))
    vis = np.asarray(run.radii) > 0
    T = np.asarray(run.transMat)[vis].astype(f32)
    centre = np.asarray(run.center)[vis].astype(f32)
    opac = sc["opacities"].numpy().reshape(-1)[vis].astype(f32)
    lo, hi = _octagon(T, centre, opac)
    return centre, T[:, 8], opac, lo, hi


def test_block_bits_on_the_bench_scene_centre_and_border_tiles(checker):
    size = 512
    centre, twz, opac, lo, hi = _scene_records(131072, size, 0)
    g = size // 16
    tiles = [(g // 2, g // 2), (g // 2 - 1, g // 2), (0, 0), (g - 1, 0), (0, g - 1), (g - 1, g - 1), (g - 1, g // 2),
             (g // 2, 0)]
    # the splats that can reach those tiles at all, and a sample of the rest
    near = np.zeros(centre.shape[0], bool)
    for tx, ty in tiles:
        near |= (np.abs(centre[:, 0] - (tx * 16 + 8)) < 64) & (np.abs(centre[:, 1] - (ty * 16 + 8)) < 64)
    pick = near | (np.arange(centre.shape[0]) % 16 == 0)
    bits = _compare(checker, _records(centre[pick], twz[pick], opac[pick], lo[pick], hi[pick]), tiles)
    # the comparison has teeth: splats touch some blocks of a tile and miss others
    assert (bits != 0).sum() > 1000
    assert ((bits != 0) & (bits != 0xFF)).sum() > 300


@pytest.mark.parametrize("x0,y0,seed", [(720, 730, 0), (700, 250, 1), (250, 740, 2)])
def test_block_bits_far_from_the_origin_and_for_faint_splats(checker, x0, y0, seed):
    P = 60000
    g = torch.Generator().manual_seed(seed)
    faint = torch.rand((P, 1), generator=g) * 0.03 + 0.0035
    barely = (1.0 / 255.0) * (1.0 + torch.rand((P, 1), generator=g) * 0.08)
    opacities = torch.where(torch.rand((P, 1), generator=g) < 0.5, faint, barely).float()
    centre, twz, opac, lo, hi = _scene_records(P, 1024, seed, opacities=opacities, scale=0.6)
    win = 64
    near = (centre[:, 0] > x0 - 16) & (centre[:, 0] < x0 + win + 16) & (centre[:, 1] > y0 - 16) & (centre[:, 1] < y0 + win + 16)
    assert near.sum() > 100
    tiles = [(tx, ty) for ty in range(y0 // 16, (y0 + win) // 16 + 1) for tx in range(x0 // 16, (x0 + win) // 16 + 1)]
    bits = _compare(checker, _records(centre[near], twz[near], opac[near], lo[near], hi[near]), tiles)
    assert ((bits != 0) & (bits != 0xFF)).sum() > 50


def test_block_bits_unbounded_empty_and_edge_octagons(checker):
    rng = np.random.default_rng(0)
    tiles = [(0, 0), (3, 5), (31, 31), (63, 1)]
    rows = []
    # unbounded (tau-ellipse crosses the camera plane) and empty (opacity < 1/255) octagons, as preprocess.cu stores them
    for cx, cy in [(8.0, 8.0), (500.0, 90.0), (-40.0, 2000.0), (1e5, -1e5)]:
        rows.append(_records(np.array([[cx, cy]], f32), np.ones(1, f32), np.ones(1, f32),
                             np.full((1, 4), -3.0e38, f32), np.full((1, 4), 3.0e38, f32)))
        rows.append(_records(np.array([[cx, cy]], f32), np.ones(1, f32), np.zeros(1, f32),
                             np.full((1, 4), 3.0e38, f32), np.full((1, 4), -3.0e38, f32)))
    # edges on the blocks' bounds: centres on pixel centres and half-pixel offsets, offsets that are small integers, so
    # cx + offset lands exactly on a block's xmin / xmax (and likewise y, x + y, x - y) for many of them
    n = 20000
    tx, ty = rng.integers(0, 64, n), rng.integers(0, 32, n)
    cx = (tx * 16 + rng.integers(-8, 24, n)).astype(f32) + rng.choice([0.0, 0.5], n).astype(f32)
    cy = (ty * 16 + rng.integers(-8, 24, n)).astype(f32) + rng.choice([0.0, 0.5], n).astype(f32)
    lo = -rng.integers(0, 12, (n, 4)).astype(f32) - rng.choice([0.0, 0.5], (n, 4)).astype(f32)
    hi = rng.integers(0, 12, (n, 4)).astype(f32) + rng.choice([0.0, 0.5], (n, 4)).astype(f32)
    # a few inverted (empty along one axis) and one-sided unbounded axes
    lo[:200, 2] = 5.0; hi[:200, 2] = -5.0
    lo[200:400, 3] = -np.inf; hi[400:600, 0] = np.inf
    rows.append(_records(np.stack([cx, cy], 1), np.ones(n, f32), np.ones(n, f32), lo, hi))
    rec = np.concatenate(rows)
    edge_tiles = sorted(set(tiles) | set(zip(tx[:64].tolist(), ty[:64].tolist())))
    bits = _compare(checker, rec, edge_tiles)
    assert (bits[:8:2] == 0xFF).all() and (bits[1:8:2] == 0).all()      # unbounded: every block; empty: none
    assert ((bits[8:] != 0) & (bits[8:] != 0xFF)).sum() > 100
