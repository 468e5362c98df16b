"""The NumPy voxel-map model (voxel_map_model.py) against the oracle's VoxelMap (oracle/orc_core.h).

On dyadic inputs (coordinates on a 2^-6 grid, power-of-two resolutions) fp32 storage and every squared distance are
exact, so the model and the oracle, which keeps fp64 points, must agree exactly. On random inputs they agree to the
storage quantum. The oracle keeps int voxel coordinates; the model skips what 21-bit keys cannot hold, so ranges are only
compared inside [-2^20, 2^20).
"""
import numpy as np
import pytest

from voxel_map_model import VoxelMapModel, pack_voxel, unpack_voxel, voxel_of

DYADIC = 1.0 / 64


def _options(b, levels, cap=0, normals=False):
    o = b.legacy_map_options(levels[0][0], levels[0][1], levels[0][2])
    o.num_resolutions = len(levels)
    for i, (res, B, md) in enumerate(levels):
        o.resolutions[i].resolution = res
        o.resolutions[i].max_num_points = B
        o.resolutions[i].min_distance_between_points = md
    o.capacity_voxels = cap
    o.select_valid_normals_direction = 1 if normals else 0
    return o


def _pair(orc, levels, cap=1024, normals=False):
    o = _options(orc, levels, cap, normals)
    return orc.voxel_map(o), VoxelMapModel.from_options(o)


def _crowded(rng, n_per_voxel, res, spread, dyadic=True):
    """points of a few voxels, interleaved in input order: n_per_voxel[k] candidates in voxel (k, k, 2k)"""
    pts = []
    for k, n in enumerate(n_per_voxel):
        base = np.array([k, k, 2 * k], dtype=np.float64) * res
        p = base + rng.uniform(0, spread * res, size=(n, 3))
        pts.append(p)
    p = np.concatenate(pts)
    p = p[rng.permutation(len(p))]
    return np.round(p / DYADIC) * DYADIC if dyadic else p


def _assert_exact(mo, model, levels):
    for lvl in range(levels):
        xo, vo = mo.export(lvl)
        xm, vm = model.export(lvl)
        assert mo.num_points(lvl) == model.levels[lvl].num_points
        assert mo.num_voxels(lvl) == model.levels[lvl].num_voxels
        assert np.array_equal(vo, vm)
        assert np.array_equal(xo, xm)


@pytest.mark.parametrize("B", [1, 20, 64])
@pytest.mark.parametrize("min_dist", [0.0, 0.25])
def test_dyadic_crowded_voxels_agree_exactly(orc, B, min_dist):
    rng = np.random.default_rng(B * 7 + int(min_dist * 4))
    levels = [(1.0, B, min_dist), (0.5, max(1, B // 2), min_dist / 2)]
    mo, model = _pair(orc, levels)
    for counts in ([1, 31, 32, 33], [511, 512, 513], [4096, 3]):
        pts = _crowded(rng, counts, 1.0, 0.99)
        mo.insert(pts)
        model.insert(pts)
        _assert_exact(mo, model, 2)


def test_dyadic_duplicates_and_distance_boundary(orc):
    mo, model = _pair(orc, [(1.0, 64, 0.25)])
    base = np.array([0.5, 0.5, 0.5])
    pts = np.array([base, base, base + [0.25, 0, 0], base + [0.25 + DYADIC, 0, 0], base - [0, 0.25 + DYADIC, 0]])
    mo.insert(pts)
    model.insert(pts)
    _assert_exact(mo, model, 1)
    # the first point, then the one at exactly min_dist is rejected, min_dist + 2^-6 accepted twice
    assert model.levels[0].num_points == 3
    mo0, model0 = _pair(orc, [(1.0, 64, 0.0)])
    dup = np.repeat(base[None], 10, axis=0)
    mo0.insert(dup)
    model0.insert(dup)
    _assert_exact(mo0, model0, 1)
    assert model0.levels[0].num_points == 1


def test_dyadic_eviction_and_reinsertion_agree_exactly(orc):
    rng = np.random.default_rng(5)
    mo, model = _pair(orc, [(1.0, 20, 0.25), (0.5, 8, 0.125)])
    pts = np.round(rng.uniform(-40, 40, size=(6000, 3)) / DYADIC) * DYADIC
    mo.insert(pts)
    model.insert(pts)
    _assert_exact(mo, model, 2)
    # a voxel whose first point lies exactly at the distance stays
    first = model.export(0)[0][0]
    loc = first + np.array([3.0, 4.0, 0.0])
    for location, distance in ((loc, 5.0), ((2.0, -3.0, 1.0), 20.0)):
        mo.remove_far(location, distance)
        model.remove_far(location, distance)
        _assert_exact(mo, model, 2)
        if distance == 5.0:
            assert any(np.array_equal(p, first) for p in model.export(0)[0])
            assert model.levels[0].num_voxels < 10
    mo.insert(pts[::2])
    model.insert(pts[::2])
    _assert_exact(mo, model, 2)


def test_random_inputs_agree_to_the_storage_quantum(orc):
    rng = np.random.default_rng(17)
    levels = [(0.7, 20, 0.05), (1.3, 33, 0.1)]
    mo, model = _pair(orc, levels, cap=1 << 12)
    for k in range(3):
        pts = rng.uniform(-25, 25, size=(8000, 3))
        pts[: 4000, 2] = rng.normal(0.0, 0.02, size=4000)
        mo.insert(pts)
        model.insert(pts)
        if k == 1:
            mo.remove_far((3.0, 1.0, 0.0), 18.0)
            model.remove_far((3.0, 1.0, 0.0), 18.0)
        for lvl, (res, _, _) in enumerate(levels):
            xo, vo = mo.export(lvl)
            xm, vm = model.export(lvl)
            assert np.array_equal(vo, vm)
            # fp32 offsets inside a voxel of side res: half an ulp of res
            assert np.abs(xo - xm).max() <= np.spacing(np.float32(res)) / 2


def test_range_edges(orc):
    res = 0.5
    mo, model = _pair(orc, [(res, 20, 0.0)])
    lo, hi = -(1 << 20), (1 << 20) - 1
    inside = []
    for axis in range(3):
        for v in (lo, hi):
            p = np.full(3, 0.25)
            p[axis] = v * res + (0.25 if v > 0 else -0.25)
            inside.append(p)
    inside = np.array(inside)
    mo.insert(inside)
    model.insert(inside)
    _assert_exact(mo, model, 1)
    assert model.levels[0].num_voxels == len(inside)
    # beyond the range: skipped by the model (the oracle's int voxels would keep them)
    for p in ([(1 << 20) * res + 0.25, 0, 0], [0, 0, -((1 << 20) + 1) * res - 0.25], [-((1 << 20) + 1) * res - 0.25] * 3,
              [np.nan, 0, 0], [np.inf, 0, 0], [1e300, 0, 0]):
        assert voxel_of(np.array(p, dtype=np.float64), res) is None
    model.insert(np.array([[(1 << 20) * res + 0.25, 0, 0]]))
    assert model.levels[0].num_voxels == len(inside)
    for v in ((lo, lo, lo), (hi, hi, hi), (0, 4, hi), (lo, 0, hi)):
        assert unpack_voxel(pack_voxel(v)) == v
    assert pack_voxel((hi, hi, hi)) < (1 << 64) - 2     # no in-range key is kEmptyKey or kTombKey
