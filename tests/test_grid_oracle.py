"""The CPU restatement of slam::SamplePointsInGrid (tests/oracle_grid) against an independent NumPy statement, the
reference's own unit case (test_A_grid_sampling.cxx), and the ctypes layouts of the grid-sampling / world-cloud ABI."""
import ctypes as C

import numpy as np
import pytest

from grid_numpy import sample_points_in_grid as np_sample
from oracle_grid_lib import grid_oracle


def _cloud(n, seed, scale=3.0):
    rng = np.random.default_rng(seed)
    return rng.uniform(-scale, scale, (n, 3))


@pytest.mark.parametrize("n", [0, 1, 2, 1000, 100_000])
@pytest.mark.parametrize("npv", [0, 1, 2, 5])
def test_oracle_matches_numpy(n, npv):
    xyz = _cloud(n, 7 + n)
    got = grid_oracle().sample_points_in_grid(xyz, 0.5, npv, -1)
    np.testing.assert_array_equal(got, np_sample(xyz, 0.5, npv, -1))


@pytest.mark.parametrize("max_num_points", [-7, -1, 0, 1, 37, 10 ** 9])
def test_oracle_max_num_points(max_num_points):
    xyz = _cloud(5000, 3)
    got = grid_oracle().sample_points_in_grid(xyz, 0.3, 2, max_num_points)
    full = np_sample(xyz, 0.3, 2, -1)
    exp = full if max_num_points < 0 else full[:max_num_points + 1]
    np.testing.assert_array_equal(got, exp)
    if max_num_points == 0:
        assert len(got) == 1   # size() > max is tested before each push: max 0 returns one point


def test_truncated_voxel_zero_and_faces():
    # int(p / s) truncates toward zero: (-0.9, 0.9) share voxel 0; -1.0 and 1.0 lie exactly on faces of voxels -1 and 1
    xyz = np.array([[0.9, 0, 0], [-0.9, 0, 0], [-1.0, 0, 0], [1.0, 0, 0], [-1.5, 0, 0], [1.999999, 0, 0],
                    [2.0, 0, 0], [-2.0, -0.5, 0.5], [0.0, -0.0, 0.0]])
    got = grid_oracle().sample_points_in_grid(xyz, 1.0, 1, -1)
    np.testing.assert_array_equal(got, [0, 2, 3, 6, 7])
    np.testing.assert_array_equal(got, np_sample(xyz, 1.0, 1, -1))
    rng = np.random.default_rng(11)
    faces = rng.integers(-50, 50, (20000, 3)) * 0.1          # on (or within an ulp of) the faces of a 0.1 grid
    for npv in (1, 3):
        np.testing.assert_array_equal(grid_oracle().sample_points_in_grid(faces, 0.1, npv, -1),
                                      np_sample(faces, 0.1, npv, -1))


def test_rejections_are_skipped_but_numbered():
    xyz = _cloud(2000, 5)
    xyz[3] = [np.nan, 0, 0]
    xyz[10] = [0, np.inf, 0]
    xyz[20] = [0, 0, 2.0 ** 20 * 0.5]          # voxel coordinate 2^20 at 0.5: outside [-2^20, 2^20)
    xyz[21] = [-(2.0 ** 20) * 0.5, 0, 0]       # -2^20: inside
    got = grid_oracle().sample_points_in_grid(xyz, 0.5, 2, -1)
    assert 3 not in got and 10 not in got and 20 not in got and 21 in got
    np.testing.assert_array_equal(got, np_sample(xyz, 0.5, 2, -1))


def test_reference_unit_case():
    # test_A_grid_sampling.cxx: 1000 points |Random()| in [0, 1]^3, grid 0.34, one per voxel: no more points than input
    xyz = np.abs(np.random.default_rng(0).uniform(-1, 1, (1000, 3)))
    got = grid_oracle().sample_points_in_grid(xyz, 0.34, 1, -1)
    assert len(got) <= 1000 and len(got) == 27   # [0, 1] spans voxels 0..2 on each axis
    np.testing.assert_array_equal(got, np_sample(xyz, 0.34, 1, -1))


def test_refusals():
    b = grid_oracle()
    for g in (0.0, -1.0, np.nan, np.inf):
        with pytest.raises(Exception):
            b.sample_points_in_grid(np.zeros((2, 3)), g)
    with pytest.raises(Exception):
        b.sample_points_in_grid(np.zeros((2, 3)), 1.0, 65)


def test_ctypes_layouts():
    from ct_icp_b200 import _abi as abi
    import ct_icp_b200
    assert C.sizeof(abi.GridSamplingOptions) == 24 and abi.GridSamplingOptions.max_num_points.offset == 16
    assert C.sizeof(abi.WorldCloudStats) == 32
    eng = ct_icp_b200.engine()
    assert eng.fn("abi_sizeof")(b"cticp_grid_sampling_options") == C.sizeof(abi.GridSamplingOptions)
    assert eng.fn("abi_sizeof")(b"cticp_world_cloud_stats") == C.sizeof(abi.WorldCloudStats)
    o = abi.GridSamplingOptions()
    eng.fn("default_grid_sampling_options")(C.byref(o))
    assert (o.grid_size, o.num_points_per_voxel, o.max_num_points) == (1.0, 1, -1)
