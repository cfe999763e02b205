"""CPU study: phase-1 work of the blend backward when the groups come from the octagon cull (today) vs from the
forward's contributing pairs (replay).  128x128 crop of the north-star view, 8x4 blocks, groups of 16, index order."""
import os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_cull_invariant as t
from lara_b200 import scene as S
from oracle import oracle as O

f32 = np.float32
P, H, W = 131072, 512, 512
sc = S.scene(P, 0)
cam = S.cameras(8, H, W, 0)[0]
run = O.run_scene(sc, cam, torch.ones(3))
vis = np.asarray(run.radii) > 0
T = np.asarray(run.transMat).astype(f32); c = np.asarray(run.center).astype(f32); rad = np.asarray(run.radii)
o = sc["opacities"].numpy().reshape(-1).astype(f32)
x0 = y0 = 192; n = 128
touch = vis & (o >= 1 / 255.0) & (c[:, 0] + rad > x0) & (c[:, 0] - rad < x0 + n) & (c[:, 1] + rad > y0) & (c[:, 1] - rad < y0 + n)
idx = np.nonzero(touch)[0]
nb = (n // 4) * (n // 8)
oct_rows = [[] for _ in range(nb)]
val_rows = [[] for _ in range(nb)]
for s in range(0, len(idx), 1500):
    ii = idx[s:s + 1500]
    Ts = T[ii].copy(); cs = c[ii].copy()
    Ts[:, 0:3] -= f32(x0) * Ts[:, 6:9]; Ts[:, 3:6] -= f32(y0) * Ts[:, 6:9]
    cs[:, 0] -= x0; cs[:, 1] -= y0
    valid, px, py = t._valid_pairs(Ts, cs, o[ii], n, n)
    lo, hi = t._octagon(Ts, cs, o[ii])
    cc = lambda a: a[:, None, None]
    coords = [px - cc(cs[:, 0]), py - cc(cs[:, 1]), (px + py) - cc(cs[:, 0] + cs[:, 1]), (px - py) - cc(cs[:, 0] - cs[:, 1])]
    octa = np.ones(valid.shape, bool)
    for k in range(4):
        octa &= (coords[k] >= cc(lo[:, k])) & (coords[k] <= cc(hi[:, k]))
    rs = lambda a: a.reshape(len(ii), n // 4, 4, n // 8, 8).transpose(0, 1, 3, 2, 4).reshape(len(ii), nb, 32)
    op, vp = rs(octa), rs(valid)
    for gi, bi in zip(*np.nonzero(op.any(2))):
        oct_rows[bi].append((op[gi, bi], vp[gi, bi]))
    for gi, bi in zip(*np.nonzero(vp.any(2))):
        val_rows[bi].append(vp[gi, bi])
G = 16
to = go = tv = gv = pairs = octpairs = 0
for rows in oct_rows:
    for k in range(0, len(rows), G):
        m = np.stack([r[0] for r in rows[k:k + G]])
        to += int(m.sum(0).max()); go += 1; octpairs += int(m.sum())
for rows in val_rows:
    for k in range(0, len(rows), G):
        m = np.stack(rows[k:k + G])
        tv += int(m.sum(0).max()); gv += 1; pairs += int(m.sum())
print(f"entries per block: octagon-hit {sum(map(len, oct_rows)) / nb:.1f}, contributing {sum(map(len, val_rows)) / nb:.1f}")
print(f"pairs: octagon {octpairs}, valid {pairs} ({pairs / octpairs:.2f})")
print(f"groups of {G}: octagon {go}, replay {gv} ({gv / go:.2f})")
print(f"phase-1 trips: octagon {to} ({octpairs / to:.1f} lanes busy/trip, {pairs / to:.1f} useful), replay {tv} ({pairs / tv:.1f} useful/trip), ratio {tv / to:.2f}")
