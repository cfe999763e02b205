"""The per-warp walk of the blend backward (render_bwd.cu), replayed lane by lane on the CPU.

Each warp walks its own 8x4 block's list positions back to front from its own deepest contributor, 128 per step
(lane l reads positions wmax-1-(128 b + 32 k + l), k = 0..3), ballot-compacts the non-zero mask words into its queue
behind the entries carried from the last step, processes every full 32-entry chunk (two 16-entry groups), and moves
the rest to the front of the queue; its last step processes all that is left.  Phase 1 finds the median contributor by
comparing list positions.  Checked: every (block, contributing position) is taken exactly once and back to front, every
group but the warp's last is full, each pixel's median position is met exactly once, and the queue never overflows."""
import numpy as np
import pytest

WINDOW, CHUNK, GROUP = 128, 32, 16
QUEUE = CHUNK - 1 + WINDOW


def walk(masks, wmax):
    """masks: the block's u32 mask per list position.  Returns the groups as lists of (position, mask)."""
    steps = (wmax + WINDOW - 1) // WINDOW
    queue, groups = [], []
    for b in range(steps):
        for k in range(WINDOW // 32):
            mk = [0] * 32
            for lane in range(32):
                pos = wmax - 1 - (b * WINDOW + k * 32 + lane)
                mk[lane] = int(masks[pos]) if pos >= 0 else 0
            hits = [lane for lane in range(32) if mk[lane]]                  # ballot, prefix popc per lane
            for lane in hits:
                queue.append((wmax - 1 - (b * WINDOW + k * 32 + lane), mk[lane]))
        assert len(queue) <= QUEUE
        nh = len(queue) if b == steps - 1 else len(queue) & ~(CHUNK - 1)
        for g0 in range(0, nh, CHUNK):
            for sub in range(2):
                gbase = g0 + sub * GROUP
                if gbase >= nh:
                    break
                groups.append(queue[gbase:min(gbase + GROUP, nh)])
        queue = queue[nh:]                                                   # the carry
    assert not queue
    return groups


def check(masks, n_contrib, median):
    """n_contrib / median: per pixel of the block (32), the forward's last and median contributor counts."""
    wmax = max(n_contrib)
    groups = walk(masks, wmax)
    taken = [p for g in groups for p, _ in g]
    want = [p for p in range(wmax - 1, -1, -1) if masks[p]]
    assert taken == want, "an entry lost, repeated or out of back-to-front order"
    assert all(len(g) == GROUP for g in groups[:-1]), "a group other than the warp's last is partial"
    for px in range(32):
        pos_median = median[px] - 1
        hits = [p for g in groups for p, m in g if p == pos_median and (m >> px) & 1]
        blended = median[px] > 0 and (masks[median[px] - 1] >> px) & 1
        assert len(hits) == (1 if blended else 0), "median contributor not met exactly once"
    return groups


def random_block(rng, n, density, wmax=None):
    masks = np.zeros(max(n, 1), np.int64)
    for p in range(n):
        if rng.random() < density:
            masks[p] = int(rng.integers(1, 1 << 32))
    wmax = n if wmax is None else wmax
    masks[wmax:] = 0                                                         # not recorded at or behind the warp's depth
    nz = [p for p in range(wmax) if masks[p]]
    n_contrib = [0] * 32
    median = [0] * 32
    for px in range(32):
        mine = [p for p in nz if (masks[p] >> px) & 1]
        n_contrib[px] = mine[-1] + 1 if mine else 0
        median[px] = mine[len(mine) // 2] + 1 if mine else 0
    if nz:
        n_contrib[0] = max(n_contrib[0], wmax)                               # the block's deepest contributor
    return masks, n_contrib, median


def test_random_blocks():
    rng = np.random.default_rng(3)
    for trial in range(300):
        n = int(rng.integers(0, 700))
        masks, nc, med = random_block(rng, n, float(rng.choice([0.02, 0.2, 0.5, 1.0])))
        check(masks, nc, med)


def test_empty_warp():
    masks = np.zeros(64, np.int64)
    assert check(masks, [0] * 32, [0] * 32) == []


def test_warp_deeper_than_its_cta():
    # one warp of a CTA walks 1000 positions, another 40: each from its own depth, with its own number of steps
    rng = np.random.default_rng(5)
    deep = random_block(rng, 1000, 0.3)
    shallow = random_block(rng, 40, 0.3)
    g_deep, g_shallow = check(*deep), check(*shallow)
    assert sum(map(len, g_deep)) > 10 * sum(map(len, g_shallow))


@pytest.mark.parametrize("n", [QUEUE + 1, 4 * WINDOW + 17, 3000])
def test_list_longer_than_the_queue(n):
    # every position contributes: each step brings 128 entries behind up to 31 carried ones
    masks = np.full(n, 0xffffffff, np.int64)
    nc = [n] * 32
    med = [n // 2 + 1] * 32
    groups = check(masks, nc, med)
    assert len(groups) == -(-n // GROUP)


def test_carry_at_every_step():
    # 33 entries per step: one full chunk and one carried entry each time
    n = 5 * WINDOW
    masks = np.zeros(n, np.int64)
    for b in range(5):
        for j in range(33):
            masks[n - 1 - (b * WINDOW + 3 * j)] = 1 << (j % 32)
    wmax = n
    nc = [0] * 32
    nc[0] = wmax
    check(masks, nc, [0] * 32)
