"""Host model of the warp-windowed decoupled look-back (ct_icp_b200/csrc/frame_pipeline.cu: tile_lookback).

A tile publishes its count (status 1), then one warp reads the 32 descriptors before a window end, lane j tile
end - 32 + j; a lane whose descriptor is still unpublished (status 0) reloads it. If some lane holds an inclusive prefix
(status 2), the tile's prefix gains the highest such lane's value and the counts of the lanes above it; otherwise it gains
all 32 counts and the window moves back by 32. The tile then publishes its inclusive prefix (status 2).

The model interleaves every lane load of every tile under random schedules (all tiles started at once, as in the
cooperative k_sample_fused, or started in ticket order, as in k_grid_select), so a window can mix descriptors read before
and after a neighbour published. Every prefix must be the exclusive scan of the counts. A lockstep schedule checks the
number of dependent window trips: at most ceil(t / 32) for tile t, and 3 for the last of 128 tiles (a 130k-point scan in
selection 1 of the fused sampler), where the walk of one descriptor per trip took 16.
"""
import math
import random

import numpy as np
import pytest


def lookback_steps(tile, count, desc, result, rng):
    """one tile's look-back as a generator: yields between any two descriptor accesses"""
    if tile == 0:
        desc[0] = (2, count)
        result[0] = 0
        return
    desc[tile] = (1, count)
    yield
    before, end = 0, tile
    while True:
        window = [None] * 32
        lanes = list(range(32))
        rng.shuffle(lanes)                      # the lanes' loads land in any order
        for lane in lanes:
            t = end - 32 + lane
            if t < 0:
                window[lane] = (2, 0)
                continue
            while True:
                window[lane] = desc[t]
                yield
                if window[lane][0] != 0:
                    break
        inclusive = [lane for lane in range(32) if window[lane][0] == 2]
        if inclusive:
            hi = max(inclusive)
            before += sum(window[lane][1] for lane in range(hi, 32))
            break
        before += sum(v for _, v in window)
        end -= 32
    desc[tile] = (2, before + count)
    result[tile] = before


def run(counts, rng, ticket_order):
    tiles = len(counts)
    desc = [(0, 0)] * tiles
    result = {}
    pending = list(range(tiles))
    if not ticket_order:
        rng.shuffle(pending)
    running = []
    while pending or running:
        # ticket order: a tile starts only after every tile before it has started
        if pending and (not running or rng.random() < 0.3):
            t = pending.pop(0)
            running.append(lookback_steps(t, int(counts[t]), desc, result, rng))
            continue
        g = rng.choice(running)
        try:
            next(g)
        except StopIteration:
            running.remove(g)
    return result


@pytest.mark.parametrize("ticket_order", [False, True])
def test_windowed_lookback_prefixes_are_the_exclusive_scan(ticket_order):
    rng = random.Random(3 + ticket_order)
    nprng = np.random.default_rng(5 + ticket_order)
    for tiles in (1, 2, 31, 32, 33, 64, 65, 100, 128, 300):
        for _ in range(3):
            counts = nprng.integers(0, 1025, size=tiles)
            counts[nprng.random(tiles) < 0.2] = 0        # empty tiles
            result = run(counts, rng, ticket_order)
            excl = np.concatenate([[0], np.cumsum(counts)[:-1]])
            assert [result[t] for t in range(tiles)] == excl.tolist()


def lockstep_trips(tiles, window):
    """every tile has published its count; then each round every unfinished tile reads one window (all of it as the
    round starts), and the tiles that met an inclusive prefix publish theirs at the end of the round. -> rounds per tile"""
    status = [2] + [1] * (tiles - 1)
    done = [1] + [0] * (tiles - 1)
    end = list(range(tiles))
    rounds = [0] * tiles
    r = 0
    while not all(done):
        r += 1
        finished = []
        for t in range(1, tiles):
            if done[t]:
                continue
            lo = max(0, end[t] - window)
            if any(status[s] == 2 for s in range(lo, end[t])):
                finished.append(t)
                rounds[t] = r
            else:
                end[t] = lo
        for t in finished:
            status[t] = 2
            done[t] = 1
    return rounds


@pytest.mark.parametrize("tiles,serial_trips,window_trips", [(12, 5, 1), (128, 16, 3), (1000, 45, 8), (4096, 90, 16)])
def test_windowed_lookback_trips(tiles, serial_trips, window_trips):
    rounds = lockstep_trips(tiles, 32)
    for t in range(1, tiles):
        assert rounds[t] <= math.ceil(t / 32)
    assert max(rounds) == window_trips
    # the one-descriptor walk the window replaces: tile t is done at the first trip s with T(t - s) < s, so ~sqrt(2t)
    assert max(lockstep_trips(tiles, 1)) == serial_trips
