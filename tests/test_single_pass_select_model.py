"""Host model of the single-pass grid selection (ct_icp_b200/csrc/frame_pipeline.cu: select_tile_dev, tile_lookback,
k_sample_fused, k_grid_select).

Claim files each point's voxel slot (and, under the first permutation, its index) at its position p = priority. A tile of
1024 positions then tests its winners (the bid (p << 32 | i) is the minimum of its voxel), publishes its count, and finds the
number of winners before it by decoupled look-back over the tiles before it. The model runs the tiles as interleaved steps
under random schedules (all tiles started at once, as in the cooperative launch, or started in ticket order, as in the
standalone kernel), over several frames whose scan sizes jump, with the descriptor arrays reused and cleared the way the
fused sampler clears them. Every tile's prefix must be numpy.cumsum's and every output the order contract's (DESIGN §4):
winners = first point per voxel in permuted order, output in ascending priority, then scattered by the second permutation.
"""
import random

import numpy as np
import pytest

TILE = 1024
MAX_TILES = 4096


def claim(keys, prio):
    """-> slot_at, src by position; vals per voxel (min bid)"""
    n = len(keys)
    slot_at = np.empty(n, dtype=np.int64)
    src = np.empty(n, dtype=np.int64)
    vals = {}
    for i in range(n):
        p = int(prio[i])
        bid = (p << 32) | i
        vals[keys[i]] = min(vals.get(keys[i], bid), bid)
        slot_at[p] = keys[i]
        src[p] = i
    return slot_at, src, vals


def tile_steps(tile, n, slot_at, src, vals, desc, result):
    """one tile as a generator: yields while waiting on a predecessor that has not published yet"""
    lo, hi = tile * TILE, min(n, (tile + 1) * TILE)
    win = [int(src[p]) for p in range(lo, hi) if vals[slot_at[p]] == ((p << 32) | int(src[p]))]
    count = len(win)
    yield
    if tile == 0:
        desc[0] = (2, count)
        before = 0
    else:
        desc[tile] = (1, count)
        yield
        before, t = 0, tile - 1
        while True:
            status, value = desc[t]
            if status == 0:
                yield
                continue
            before += value
            if status == 2:
                break
            t -= 1
            yield
        desc[tile] = (2, before + count)
    result[tile] = (before, win)


def run_selection(n, slot_at, src, vals, desc, rng, ticket_order):
    tiles = (n + TILE - 1) // TILE
    for t in range(tiles):
        assert desc[t] == (0, 0), "descriptor %d not clean" % t
    result = {}
    pending = list(range(tiles))
    if not ticket_order:
        rng.shuffle(pending)
    running = []
    while pending or running:
        # ticket order: a tile starts only after every tile before it has started (its CTA is then resident)
        if pending and (not running or rng.random() < 0.5):
            t = pending.pop(0)
            running.append(tile_steps(t, n, slot_at, src, vals, desc, result))
            continue
        g = rng.choice(running)
        try:
            next(g)
        except StopIteration:
            running.remove(g)
    counts = np.array([len(result[t][1]) for t in range(tiles)], dtype=np.int64)
    excl = np.concatenate([[0], np.cumsum(counts)[:-1]]) if tiles else counts
    for t in range(tiles):
        assert result[t][0] == excl[t]
    out = [i for t in range(tiles) for i in result[t][1]]
    return out


def reference_winners(keys, prio):
    best = {}
    for i, k in enumerate(keys):
        if k not in best or prio[i] < prio[best[k]]:
            best[k] = i
    return sorted(best.values(), key=lambda i: prio[i])


@pytest.mark.parametrize("ticket_order", [False, True])
def test_single_pass_selection_matches_cumsum_and_order_contract(ticket_order):
    rng = random.Random(7 + ticket_order)
    nprng = np.random.default_rng(11 + ticket_order)
    desc1 = [(0, 0)] * MAX_TILES
    desc2 = [(0, 0)] * MAX_TILES
    for n in (5000, 1, 1024, 1025, 9000, 0, 3000, 12000, 2048):
        # selection 1: N points, voxel keys with many repeats, first permutation
        keys = nprng.integers(0, max(1, n // 3), size=n).tolist()
        perm1 = nprng.permutation(n)
        tiles1 = (n + TILE - 1) // TILE
        for t in range(tiles1):          # phase 1 clears selection 2's descriptors (F <= N)
            desc2[t] = (0, 0)
        slot_at, src, vals = claim(keys, perm1)
        win = run_selection(n, slot_at, src, vals, desc1, rng, ticket_order)
        assert win == reference_winners(keys, perm1)
        # the second shuffle, then selection 2 on the frame (priority = frame index, no permutation)
        F = len(win)
        perm2 = nprng.permutation(F)
        frame = [None] * F
        for k, i in enumerate(win):
            frame[perm2[k]] = i
        keys2 = [keys[i] // 4 for i in frame]
        slot_at2, src2, vals2 = claim(keys2, np.arange(F))
        kp = run_selection(F, slot_at2, src2, vals2, desc2, rng, ticket_order)
        assert kp == reference_winners(keys2, np.arange(F))
        for t in range(tiles1):          # phase 4 leaves selection 1's descriptors clean for the next frame
            desc1[t] = (0, 0)
