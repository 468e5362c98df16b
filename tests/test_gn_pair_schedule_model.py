"""Host model of the paired tile schedule of k_gn_persistent (ct_icp_b200/csrc/icp_gn.cu: gn_pairs_apply, gn_pair_schedule,
gn_gather_tiles): from the second iteration on, a gather CTA whose range holds more keypoints than warps but at most two
per warp gives every warp one tile — the heaviest keypoints of the last iteration alone, the others in pairs, heaviest with
lightest. Restated one-to-one (same rank rule, same slot arithmetic); the one-keypoint-per-grab schedule it replaces there
is the model of test_gn_loop_model.py."""
import itertools
import random

import numpy as np
import pytest

from test_gn_loop_model import K_GATHER_WARPS, K_ROW_PARTS, cta_gather, tile_width

NO_KEYPOINT = 0xff   # kNoKeypoint


def pairs_apply(span):
    """gn_pairs_apply"""
    return K_GATHER_WARPS > 1 and 2 * K_GATHER_WARPS <= 32 and K_GATHER_WARPS < span <= 2 * K_GATHER_WARPS


def pair_schedule(cost):
    """gn_pair_schedule: cost[r] of the range's keypoints r = 0..n-1 -> pair[w] = [first, second] per warp. Lane r computes
    its rank (heaviest first, lower index first among equals) and writes its slot."""
    n = len(cost)
    pair = [[None, None] for _ in range(K_GATHER_WARPS)]
    singles, pairs = 2 * K_GATHER_WARPS - n, n - K_GATHER_WARPS
    for lane in range(n):
        c = cost[lane]
        rank = sum(1 for j in range(n) if cost[j] > c or (cost[j] == c and j < lane))
        if rank < singles:
            pair[rank] = [lane, NO_KEYPOINT]
        elif rank < singles + pairs:
            pair[rank][0] = lane
        else:
            pair[singles + (n - 1 - rank)][1] = lane
    return pair


def tiles_of(pair):
    """gn_gather_tiles with a schedule: warp w's one tile, (wt, rows)"""
    out = []
    for a, b in pair:
        wt = 1 if b == NO_KEYPOINT else 2
        out.append([a] if wt == 1 else [a, b])
    return out


def reduce_rows(table, n):
    """gn_cta_reduce_rows (one chunk)"""
    parts = []
    for part in range(K_ROW_PARTS):
        s = 0.0
        for r in range(part, n, K_ROW_PARTS):
            s += table[r]
        parts.append(s)
    s = parts[0]
    for q in range(1, K_ROW_PARTS):
        s += parts[q]
    return s


@pytest.mark.parametrize("span", [16, 17, 24, 31, 32, 33])
def test_every_keypoint_once(span):
    rng = np.random.default_rng(span)
    if not pairs_apply(span):
        # 16 and 33: the grab schedule as before (one keypoint per grab up to 32, then wider tiles)
        assert span in (16, 33) and tile_width(span) == (1 if span <= 32 else 3)
        visits, _ = cta_gather(0, span, random.Random(span), lambda k: 1.0)
        assert sorted(visits) == list(range(span)) and set(visits.values()) == {1}
        return
    for trial in range(50):
        cost = [int(x) for x in rng.integers(0, 40 if trial % 2 else 4000, size=span)]
        pair = pair_schedule(cost)
        assert all(p[0] is not None and p[1] is not None for p in pair)   # every warp's tile is complete
        rows = [r for t in tiles_of(pair) for r in t]
        assert sorted(rows) == list(range(span))
        assert sum(len(t) == 2 for t in tiles_of(pair)) == span - K_GATHER_WARPS


def test_grab_schedule_unchanged_outside_the_paired_spans():
    assert [pairs_apply(s) for s in (0, 1, 15, 16, 17, 32, 33, 200, 256, 300)] == \
        [False, False, False, False, True, True, False, False, False, False]
    for c_lo, c_hi in ((0, 300), (5, 600)):          # ranges of more than kRowCap keypoints go in chunks, as before
        visits, _ = cta_gather(c_lo, c_hi, random.Random(c_hi), lambda k: 1.0)
        assert sorted(visits) == list(range(c_lo, c_hi)) and set(visits.values()) == {1}


@pytest.mark.parametrize("span", [17, 18, 20, 24, 31, 32])
def test_schedule_is_a_function_of_the_costs(span):
    rng = np.random.default_rng(100 + span)
    cost = [int(x) for x in rng.integers(0, 6, size=span)]   # many ties
    pair = pair_schedule(cost)
    assert pair == pair_schedule(list(cost))
    # the order heaviest first, lower index first among equals: singles in that order, then the pairs
    order = sorted(range(span), key=lambda r: (-cost[r], r))
    singles = 2 * K_GATHER_WARPS - span
    assert [p[0] for p in pair[:singles]] == order[:singles]
    rest = order[singles:]
    assert [tuple(p) for p in pair[singles:]] == [(rest[m], rest[-1 - m]) for m in range(span - K_GATHER_WARPS)]
    # all costs equal: the index order alone decides
    flat = pair_schedule([7] * span)
    assert [p[0] for p in flat[:singles]] == list(range(singles))


def _matchings(items):
    """every split of `items` into pairs"""
    if not items:
        yield []
        return
    first, rest = items[0], items[1:]
    for i, partner in enumerate(rest):
        for m in _matchings(rest[:i] + rest[i + 1:]):
            yield [(first, partner)] + m


@pytest.mark.parametrize("span", [17, 18])
def test_pairing_minimises_the_largest_tile(span):
    """with a tile's cost the sum of its keypoints' costs, no split into singles and pairs has a smaller maximum (brute
    force over every choice of the paired keypoints and every pairing of them)"""
    rng = np.random.default_rng(7 * span)
    npairs = span - K_GATHER_WARPS
    for _ in range(3):
        cost = [int(x) for x in rng.integers(1, 100, size=span)]
        got = max(sum(cost[r] for r in t) for t in tiles_of(pair_schedule(cost)))
        best = None
        for paired in itertools.combinations(range(span), 2 * npairs):
            solo = max(cost[r] for r in range(span) if r not in paired)
            for m in _matchings(list(paired)):
                worst = max(solo, max(cost[a] + cost[b] for a, b in m))
                best = worst if best is None else min(best, worst)
        assert got == best


@pytest.mark.parametrize("span", [17, 24, 32])
def test_reduced_row_does_not_depend_on_the_schedule(span):
    vals = np.random.default_rng(span).standard_normal(span)
    # grab schedule (random warp order)
    _, grabbed = cta_gather(0, span, random.Random(3), lambda k: float(vals[k]))
    for seed in range(5):
        cost = [int(x) for x in np.random.default_rng(seed).integers(0, 50, size=span)]
        table = {}
        for t in tiles_of(pair_schedule(cost)):
            for r in t:
                assert r not in table
                table[r] = float(vals[r])
        assert reduce_rows(table, span) == grabbed
