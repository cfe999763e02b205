"""CPU study: the blend backward's work per warp when each warp walks its own 8x4 block's contributing list entries
(compaction carried across 128-position rounds, no CTA barriers) against today's CTA-wide 128-entry rounds.

The C oracle renders the bench scene (131 072 Gaussians, seed 0, view 0, 512x512) and records, as the forward does,
one u32 pixel mask per list position and 8x4 block and each pixel's last contributor.  For every block (warp) and
half tile (4-warp CTA) of the view, or of a crop, it counts both ways

    groups          16-entry groups of compacted entries (today: cut at every 128-position round)
    phase-1 trips   the sum over groups of max-over-pixels contributing entries
    phase-2 trips   the sum over groups of C, the smallest chunk size with sum_i ceil(c_i / C) <= 32
    chunks          32-entry chunk set-ups
    walk steps      today: the CTA's 128-position rounds from the half tile's deepest contributor, every warp
                    taking part; per warp: 128-position steps from the warp's own deepest contributor
    barrier waste   today only: per round, (max over the CTA's 4 warps) - (mean) of the round's weighted cost

and weighs them with the static instruction counts of tools/sass_budget.py (DESIGN §3.3) to predict the change in
warp instructions per view.

    python tools/bwd_warp_walk_study.py                   # the full view
    python tools/bwd_warp_walk_study.py centre|border     # a 128x128 crop: the view's centre or its top-left corner
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lara_b200 import scene as S  # noqa: E402
from oracle import oracle as O  # noqa: E402

# static warp-instruction counts per part, from tools/sass_budget.py on each kernel (DESIGN §3.3).  step: a walk step
# of 128 list positions outside its chunks (rounds: mask loads, staging, two barriers, compaction; per warp: mask
# loads, compaction into the queue, the carry); gather: the per-warp walk's record fetch per 32-entry chunk
W_ROUNDS = dict(chunk=117, head=9, p1=93, between=107, p2=85, sums=20, tail=6, step=272, gather=0)
W_WARP = dict(chunk=128, head=10, p1=92, between=98, p2=85, sums=20, tail=7, step=204, gather=45)

LANE_BIT = np.uint32(1) << np.arange(32, dtype=np.uint32)


def group_counts(masks):
    """masks: [n] u32 of one warp's compacted entries, back to front.  (groups, phase-1 trips, phase-2 trips)."""
    n = len(masks)
    if n == 0:
        return 0, 0, 0
    bits = (masks[:, None] & LANE_BIT) != 0                      # [n, 32 pixels]
    ng = -(-n // 16)
    pad = np.zeros((ng * 16, 32), bool)
    pad[:n] = bits
    g = pad.reshape(ng, 16, 32)
    p1 = int(g.sum(1).max(1).sum())
    c = g.sum(2)                                                 # [ng, 16] contributing pixels per entry
    p2 = 0
    for row in c:
        row = row[row > 0]
        p2 += next(C for C in range(1, 17) if int(np.ceil(row / C).sum()) <= 32)
    return ng, p1, p2


def cost(W, ng, p1, p2, nchunks):
    return (nchunks * (W["chunk"] + W["gather"]) + ng * (W["head"] + W["between"] + W["sums"] + W["tail"])
            + p1 * W["p1"] + p2 * W["p2"])


def study(run, x0=0, y0=0, n=None):
    H, Wd = run.H, run.W
    gx = (Wd + 15) // 16
    nc = np.asarray(run.n_contrib[0]).astype(np.int64)
    ranges = np.asarray(run.ranges).astype(np.int64)
    masks = np.asarray(run.masks)
    n = n or max(H, Wd)
    t0x, t0y, t1x, t1y = x0 // 16, y0 // 16, (x0 + n) // 16, (y0 + n) // 16
    tot = {k: 0 for k in ("old_groups", "new_groups", "old_p1", "new_p1", "old_p2", "new_p2", "old_chunks", "new_chunks",
                          "old_steps", "new_steps", "entries", "waste", "old_cost", "new_cost", "blocks")}
    for ty in range(t0y, min(t1y, (H + 15) // 16)):
        for tx in range(t0x, min(t1x, gx)):
            tile = ty * gx + tx
            rx, ry = ranges[tile]
            for half in range(2):
                wm, lists = [], []
                for w in range(4):
                    gw = half * 4 + w
                    bx, by = tx * 16 + (gw & 1) * 8, ty * 16 + (gw >> 1) * 4
                    blk = nc[by:by + 4, bx:bx + 8]
                    m = int(blk.max()) if blk.size else 0
                    pos = np.arange(m - 1, -1, -1)
                    mk = masks[gw, rx + pos] if m else np.zeros(0, np.uint32)
                    wm.append(m)
                    lists.append((pos[mk != 0], mk[mk != 0]))
                n_eff = max(wm)
                rounds = -(-n_eff // 128)
                round_cost = np.zeros((max(rounds, 1), 4))
                for w in range(4):
                    pos, mk = lists[w]
                    tot["entries"] += len(mk); tot["blocks"] += 1
                    # per warp: one list, groups cut only at its end
                    ng, p1, p2 = group_counts(mk)
                    ch = -(-len(mk) // 32)
                    steps = -(-wm[w] // 128)
                    tot["new_groups"] += ng; tot["new_p1"] += p1; tot["new_p2"] += p2; tot["new_chunks"] += ch
                    tot["new_steps"] += steps
                    tot["new_cost"] += cost(W_WARP, ng, p1, p2, ch) + steps * W_WARP["step"]
                    # today: the round of list position p is (n_eff - 1 - p) // 128
                    rnd = (n_eff - 1 - pos) // 128
                    for r in range(rounds):
                        sel = mk[rnd == r]
                        ng, p1, p2 = group_counts(sel)
                        ch = -(-len(sel) // 32)
                        tot["old_groups"] += ng; tot["old_p1"] += p1; tot["old_p2"] += p2; tot["old_chunks"] += ch
                        round_cost[r, w] = cost(W_ROUNDS, ng, p1, p2, ch) + W_ROUNDS["step"]
                tot["old_steps"] += 4 * rounds
                tot["old_cost"] += float(round_cost[:rounds].sum())
                if rounds:
                    tot["waste"] += float((round_cost[:rounds].max(1) - round_cost[:rounds].mean(1)).sum())
    return tot


def main():
    where = sys.argv[1] if len(sys.argv) > 1 else "full"
    sc = S.scene(131072, 0, sh_degree=1)
    cam = S.cameras(8, 512, 512, 0)[0]
    run = O.run_scene(sc, cam, torch.ones(3))
    crop = {"full": (0, 0, None), "centre": (192, 192, 128), "border": (0, 0, 128)}[where]
    t = study(run, *crop)
    b = t["blocks"]
    print(f"{where}: {b} warp blocks, {t['entries'] / b:.1f} contributing entries per block")
    print(f"{'per warp block':24s} {'rounds':>10s} {'per-warp':>10s} {'ratio':>7s}")
    for k, name in (("groups", "groups"), ("p1", "phase-1 trips"), ("p2", "phase-2 trips"), ("chunks", "chunk set-ups"),
                    ("steps", "walk steps (128 pos.)")):
        o, nw = t["old_" + k] / b, t["new_" + k] / b
        print(f"{name:24s} {o:10.2f} {nw:10.2f} {nw / o if o else 0:7.3f}")
    o, nw = t["old_cost"] / b, t["new_cost"] / b
    print(f"{'warp instructions':24s} {o:10.0f} {nw:10.0f} {nw / o:7.3f}")
    print(f"barrier waste per warp block (weighted instructions, today): {t['waste'] / b:.0f} "
          f"({t['waste'] / t['old_cost'] * 100:.1f} % of the round form's count)")
    print(f"predicted change in warp instructions: {(nw - o) / o * 100:+.1f} % "
          f"({(t['new_cost'] - t['old_cost']) / 1e6:+.2f} M per {where})")


if __name__ == "__main__":
    main()
