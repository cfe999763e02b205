"""Phase-2 schedule of the blend backward (render_bwd.cu) in its chunk form, replayed lane by lane on the CPU.

The kernel sets up the lane allotment of both 16-entry groups of a 32-entry chunk in one pass: lane l stands for
entry l of the chunk (group l >> 4), a 4-step binary search over the chunk size C sums ceil(c_i / C) of both groups
with one warp reduction per step (each group in its own 16-bit field), a scan segmented at lane 16 gives the lanes of
every entry, and the result is kept as one packed word per lane (end | n << 8 | (C - 1) << 16).  Each group then
reads its half of those words: a lower bound finds the entry a lane works for, a binary search on popc drops the
pixels of the entry's mask that lower-ranked lanes take.  These steps are restated here with numpy in the kernel's
order and checked for what the kernel relies on: every contributing (splat, pixel) pair of both groups is taken by
exactly one lane, no lane takes more than C pairs, the lanes suffice, and C is the smallest chunk size for which they
do, in each group on its own."""
import numpy as np
import pytest


def popc(x):
    return bin(int(x) & 0xffffffff).count("1")


LANE = np.arange(32)
CAND_M = 65536 // ((LANE & 15) + 1) + 1         # lane (C - 1) of each half: the multiplier of candidate C


def chunk_schedule(masks):
    """masks: the chunk's pixel masks (1..32 entries).  Returns the packed per-lane word of the kernel."""
    ew = np.array([masks[l] if l < len(masks) else 0 for l in range(32)], dtype=np.int64)
    cnt = np.array([popc(w) for w in ew], dtype=np.int64)
    hshift = LANE & 16
    cm1 = np.zeros(32, dtype=np.int64)
    for st in (8, 4, 2, 1):
        M = np.full(32, 65536 // 8 + 1) if st == 8 else CAND_M[cm1 + st - 1]      # __shfl_sync(candM, cm1 + st - 1)
        n = ((cnt + cm1 + st - 1) * M) >> 16
        tot = int(np.sum(n << hshift)) & 0xffffffff                                # __reduce_add_sync
        mine = (tot >> hshift) & 0xffff
        cm1 = np.where(mine > 32, cm1 + st, cm1)
    n_mine = ((cnt + cm1) * CAND_M[cm1]) >> 16
    end = n_mine.copy()
    o = 1
    while o < 16:
        v = np.concatenate([end[:o], end[:-o]])                                    # __shfl_up_sync
        end = np.where((LANE & 15) >= o, end + v, end)
        o <<= 1
    assert (end < 256).all() and (n_mine < 256).all()
    return ew, end | (n_mine << 8) | (cm1 << 16)


def group_lanes(ew, sched, sub):
    """The lanes of group `sub` of the chunk: per lane (own, pixel bits taken), and the group's C."""
    hb = 16 * sub
    end = sched & 0xff
    lanes_used = end[hb + 15]
    own = np.zeros(32, dtype=np.int64)
    st = 8
    while st > 0:
        e = end[hb + own + st - 1]
        own = np.where(e <= LANE, own + st, own)
        st >>= 1
    own_s = sched[hb + own]
    own_end, own_n, C = own_s & 0xff, (own_s >> 8) & 0xff, (own_s >> 16) + 1
    word = ew[hb + own]                                                            # s_hmw[gbase + own]
    have = LANE < lanes_used
    skip = (LANE - (own_end - own_n)) * C
    out = []
    for l in range(32):
        pos, st = 0, 16
        while st > 0:
            if popc(int(word[l]) & ((1 << (pos + st)) - 1)) <= skip[l]:
                pos += st
            st >>= 1
        bits = int(word[l]) & (0xffffffff << pos) & 0xffffffff if have[l] else 0
        taken = 0
        for _ in range(min(int(C[l]), popc(bits))):                                # the lane's walk: n_take trips
            taken |= bits & -bits
            bits &= bits - 1
        out.append((int(own[l]), taken))
    assert len(set(C.tolist())) == 1, "C differs between the lanes of a group"
    return int(C[0]), out


def check(masks):
    assert 1 <= len(masks) <= 32 and all(masks), "the compacted list holds entries with a non-zero mask only"
    ew, sched = chunk_schedule(masks)
    for sub in range(2):
        words = [int(w) for w in ew[16 * sub:16 * sub + 16]]
        if 16 * sub >= len(masks):
            continue                                                               # the kernel skips an empty group
        C, lanes = group_lanes(ew, sched, sub)
        got = [0] * 16
        for own, taken in lanes:
            assert popc(taken) <= C
            assert got[own] & taken == 0, "a pair taken twice"
            got[own] |= taken
        assert got == words, "a pair lost or invented"
        cnt = np.array([popc(w) for w in words])
        need = lambda c: int(np.ceil(cnt / c).sum())
        assert need(C) <= 32 and (C == 1 or need(C - 1) > 32), "C not minimal"
        assert sum(1 for own, taken in lanes if taken) == need(C)                 # no idle lane among those in use


def random_mask(rng, kind):
    while True:
        if kind == 0:
            w = int(rng.integers(1, 1 << 32))
        elif kind == 1:
            w = int(rng.integers(0, 1 << 32)) & int(rng.integers(0, 1 << 32)) & int(rng.integers(0, 1 << 32))
        elif kind == 2:
            w = 0xffffffff if rng.random() < 0.3 else (1 << int(rng.integers(0, 32)))
        else:
            lo, n = int(rng.integers(0, 32)), int(rng.integers(1, 33))
            w = (((1 << n) - 1) << lo) & 0xffffffff
        if w:
            return w


def test_chunk_schedule_random():
    rng = np.random.default_rng(1)
    for trial in range(2000):
        kind = trial % 4
        n = 32 if trial % 3 else int(rng.integers(1, 33))                          # full and partial last chunks
        masks = [random_mask(rng, kind if rng.random() < 0.8 else int(rng.integers(0, 4))) for _ in range(n)]
        check(masks)


@pytest.mark.parametrize("masks", [
    [0xffffffff] * 32,                                  # C = 16 in both groups, two lanes per splat
    [0xffffffff] + [1] * 15 + [0xffffffff] * 16,        # groups with different C
    [0xffffffff] + [1] * 15 + [1 << 31] * 16,
    [1 << (i % 32) for i in range(32)],                 # one pair each: C = 1
    [0xffffffff],                                       # one splat alone: C = 1, 32 lanes
    [0x80000000] * 17,                                  # second group of one entry
    [0xffffffff] * 16 + [0x0000ffff] * 16,
])
def test_chunk_schedule_corner_cases(masks):
    check(masks)
