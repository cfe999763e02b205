"""Lane allotment of phase 2 of the blend backward (render_bwd.cu), replayed lane by lane on the CPU:
the warp-level steps of the kernel (shuffles, ballot, inclusive scan, lower bound, drop-the-lowest-k-bits) are
restated with numpy in the same order and checked for what the kernel relies on -- every contributing
(splat, pixel) pair is taken by exactly one lane, no lane takes more than C pairs, the lanes suffice, and C is the
smallest chunk size for which they do."""
import numpy as np
import pytest


def popc(x):
    return bin(int(x) & 0xffffffff).count("1")


def allot(words):
    """words[i] = pixel mask of splat i (16 entries).  Returns (C, per-lane (own, bits taken))."""
    lane = np.arange(32)
    p2_i, p2_h = lane & 15, lane >> 4
    candM = 65536 // (p2_i + 1) + 1
    tw = np.array([words[l] if l < 16 else 0 for l in range(32)], dtype=np.uint64)
    cnt = np.array([popc(w) for w in tw])
    if not cnt.any():
        return 0, []
    part = np.zeros(32, dtype=np.int64)
    for k in range(8):
        c = cnt[p2_h * 8 + k]                                   # __shfl_sync(cnt, p2_h * 8 + k)
        part += ((c + p2_i) * candM) >> 16
    lanes_needed = part + part[lane ^ 16]                       # __shfl_xor_sync(part, 16)
    ballot = sum(1 << l for l in range(32) if lanes_needed[l] <= 32) & 0xffff
    C = (ballot & -ballot).bit_length()                         # __ffs
    M = candM[C - 1]
    n_mine = ((cnt + C - 1) * M) >> 16
    end = n_mine.copy()
    o = 1
    while o < 16:
        v = np.concatenate([end[:o], end[:-o]])                 # __shfl_up_sync: lanes < o keep their own value
        end = np.where(lane >= o, end + v, end)
        o <<= 1
    lanes_used = end[15]
    own = np.zeros(32, dtype=np.int64)
    st = 8
    while st > 0:
        e = end[own + st - 1]
        own = np.where(e <= lane, own + st, own)
        st >>= 1
    own_end, own_n, word = end[own], n_mine[own], tw[own]
    have = lane < lanes_used
    skip = (lane - (own_end - own_n)) * C
    out = []
    for l in range(32):
        if not have[l]:
            out.append((0, 0)); continue
        pos, st = 0, 16
        while st > 0:
            below = popc(int(word[l]) & ((1 << (pos + st)) - 1))
            if below <= skip[l]:
                pos += st
            st >>= 1
        bits = int(word[l]) & (0xffffffff << pos) & 0xffffffff
        taken = 0
        for _ in range(C):                                      # the C trips of the loop: lowest bit each
            if bits == 0:
                break
            taken |= bits & -bits
            bits &= bits - 1
        out.append((int(own[l]), taken))
    return C, out


def check(words):
    C, lanes = allot(words)
    if C == 0:
        assert not any(words)
        return
    got = [0] * 16
    for own, taken in lanes:
        assert popc(taken) <= C
        assert got[own] & taken == 0, "a pair taken twice"
        got[own] |= taken
    assert got == [int(w) for w in words], "a pair lost or invented"
    cnt = np.array([popc(w) for w in words])
    need = lambda c: int(np.ceil(cnt / c).sum())
    assert need(C) <= 32 and (C == 1 or need(C - 1) > 32)
    assert sum(1 for own, taken in lanes if taken) == need(C)   # no idle lane among those in use


def test_allotment_random_groups():
    rng = np.random.default_rng(0)
    for trial in range(3000):
        kind = trial % 6
        words = []
        for i in range(16):
            if kind == 0:
                w = int(rng.integers(0, 1 << 32))
            elif kind == 1:
                w = int(rng.integers(0, 1 << 32)) & int(rng.integers(0, 1 << 32)) & int(rng.integers(0, 1 << 32))
            elif kind == 2:
                w = 0xffffffff if rng.random() < 0.3 else (1 << int(rng.integers(0, 32)))
            elif kind == 3:
                w = 0 if rng.random() < 0.6 else int(rng.integers(0, 1 << 32))
            elif kind == 4:
                lo, n = int(rng.integers(0, 32)), int(rng.integers(0, 33))
                w = (((1 << n) - 1) << lo) & 0xffffffff
            else:
                w = int(rng.integers(0, 1 << 32)) if i < int(rng.integers(0, 17)) else 0   # partial last group
            words.append(w)
        check(words)


@pytest.mark.parametrize("words", [
    [0xffffffff] * 16,                       # every splat covers the block: C = 16, two lanes each
    [0xffffffff] + [0] * 15,                 # one splat alone: C = 1, 32 lanes
    [0] * 15 + [0x80000000],                 # a single pair in the last slot
    [1 << i for i in range(16)],             # one pair each
    [0xffffffff, 1, 0xffffffff, 2] + [0] * 12,
    [0] * 16,
])
def test_allotment_corner_cases(words):
    check(words)
