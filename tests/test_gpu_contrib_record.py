"""The blend forward's contribution record (one u32 per list position and 8x4 warp block, bit l = the splat was
blended into pixel l of the block), which the blend backward replays instead of re-deriving the pairs: rebuilt here
from the forward's own state -- its homographies, centres, opacities, per-tile lists and last contributors -- with the
pair predicate of the cull-invariant test, and compared bit for bit."""
import numpy as np
import pytest
import torch

from test_cull_invariant import _valid_pairs

pytestmark = pytest.mark.gpu

f32 = np.float32


def _forward_state(sc, cam, dev):
    from lara_b200 import rasterizer as R
    from lara_b200 import scene as S
    from lara_b200.debug import unpack_state
    st = S.settings_for(cam, torch.ones(3), sc["sh_degree"], dev, R.GaussianRasterizationSettings)
    d = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in sc.items()}
    _, _, _, state = R.forward_raw(d["means3D"], d["shs"], None, d["opacities"], d["scales"], d["rotations"], None, st)
    torch.cuda.synchronize()
    u = unpack_state(state, sc["means3D"].shape[0], cam.image_height, cam.image_width)
    return {k: v.cpu().numpy() for k, v in u.items()}


def _check_record(u, H, W, tile_step=1):
    """Compares the record with the predicate at every position below each block's deepest contributor (a block's
    positions beyond it are not recorded), in every tile_step-th tile.  Returns (pairs compared, pairs blended, pairs in
    the predicate's rounding band, blocks whose deepest contributor lies before the end of their tile's list)."""
    T = u["transMat"].astype(f32)
    centre = u["means2D"].astype(f32)
    opac = u["opacity"].astype(f32)
    last = np.zeros(((H + 15) // 16 * 16, (W + 15) // 16 * 16), np.int64)
    last[:H, :W] = u["n_contrib"][0]
    rec = u["contrib_masks"].view(np.uint32)
    gx = (W + 15) // 16
    weights = (np.uint64(1) << np.arange(32, dtype=np.uint64))
    compared = blended = band_pairs = early = 0
    for t, (s, e) in enumerate(u["ranges"]):
        if e <= s or t % tile_step:
            continue
        ty, tx = divmod(t, gx)
        ids = u["point_list"][s:e]
        n = e - s
        pred = lambda T_, c_, o_: _valid_pairs(T_, c_, o_, 16, 16, tx * 16, ty * 16)[0]
        valid = pred(T[ids], centre[ids], opac[ids])
        # the predicate's rounding band: numpy rounds without fused multiply-adds (k = pix Tw - Tu cancels at
        # pixel ~400), so pairs whose verdict differs in float64, or flips with a 1e-5 relative change of the
        # opacity, may be decided otherwise by the kernels' exact sequence
        f64 = np.float64
        band = (valid != pred(T[ids].astype(f64), centre[ids].astype(f64), opac[ids].astype(f64))) | \
            (pred(T[ids], centre[ids], opac[ids] * f32(1 - 1e-5)) != pred(T[ids], centre[ids], opac[ids] * f32(1 + 1e-5)))
        lc = last[ty * 16:ty * 16 + 16, tx * 16:tx * 16 + 16]
        expected = valid & (np.arange(n)[:, None, None] < lc[None])
        # [n,16,16] -> [n, 8 blocks, 32 lanes]: block w covers columns (w&1)*8.., rows (w>>1)*4..; lane = row*8 + col
        blocks = lambda a: a.reshape(-1, 4, 4, 2, 8).transpose(0, 1, 3, 2, 4).reshape(-1, 8, 32)
        pack = lambda a: (blocks(a).astype(np.uint64) * weights).sum(-1).astype(np.uint32)
        exp_m, band_m = pack(expected), pack(band)
        wmax = blocks(lc[None])[0].max(1)                                    # [8] deepest contributor per block
        got = rec[:, s:e].T                                                  # [n, 8]
        live = np.arange(n)[:, None] < wmax[None]
        diff = (got ^ exp_m) & ~band_m & np.where(live, np.uint32(0xFFFFFFFF), np.uint32(0))
        assert not diff.any(), (f"tile {t}: {int(np.count_nonzero(diff))} (position, block) masks differ, first at "
                                f"{tuple(int(x) for x in np.argwhere(diff)[0])}")
        compared += int(live.sum()) * 32
        blended += int(np.count_nonzero(expected))
        band_pairs += int(np.count_nonzero(band))
        early += int((wmax < n).sum())
    return compared, blended, band_pairs, early


def test_contribution_record_matches_the_forward_at_the_bench_point(cuda_device):
    from lara_b200 import scene as S
    sc = S.scene(131072, 0)
    cam = S.cameras(8, 512, 512, 0)[0]
    u = _forward_state(sc, cam, cuda_device)
    compared, blended, band_pairs, _ = _check_record(u, 512, 512, tile_step=3)   # the predicate runs in numpy: 1/3 of the tiles
    assert compared > 10_000_000 and blended > 1_000_000
    assert band_pairs < 1e-4 * compared


def test_contribution_record_of_a_saturated_scene(cuda_device):
    """Opaque, large splats: most pixels saturate (T < 1e-4) early in their tile's list and whole warps stop, so the
    record ends before the list does and the saturating pairs, which the forward does not blend, must be left out."""
    from lara_b200 import scene as S
    sc = S.scene(20000, 3)
    sc["opacities"] = torch.full_like(sc["opacities"], 0.97)
    sc["scales"] = sc["scales"] * 2.5
    cam = S.cameras(3, 256, 200, 3)[1]
    u = _forward_state(sc, cam, cuda_device)
    assert (u["accum"][0] < 1e-3).mean() > 0.5
    compared, blended, band_pairs, early = _check_record(u, 256, 200)
    assert compared > 100_000 and blended > 10_000 and early > 100
    assert band_pairs < 1e-4 * compared
