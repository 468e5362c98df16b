"""The grid selections over many look-back tiles (ct_icp_b200/csrc/frame_pipeline.cu: tile_lookback's 32-descriptor
window), against the CPU oracle.

A tile of 1024 positions finds the winners before it with a window that moves back 32 tiles per trip, so the cases go up
to the 4096-tile limit of a scan (max_points_per_frame = 4 Mi points), with windows that straddle tile 0 and more
than one window per look-back:
  - the standalone selection (k_grid_select, grid_sample_indices), scans of 1 Mi + 17 and 4 Mi points;
  - both selections of the fused sampler (k_sample_fused) on a 4 Mi-point scan whose frame keeps ~2 Mi points, so the
    keypoint selection runs over ~2000 tiles as well: the scan registered twice, the second time with keypoints (the
    first frame's map, lists of ~100 candidates per voxel, is compared too).
"""
import numpy as np
import pytest

from test_gpu_parity import POS_TOL, _sequence_options

pytestmark = pytest.mark.gpu

MAX_POINTS = 4 << 20   # 4096 tiles of 1024


def _box_cloud(n, extent, height, seed):
    rng = np.random.default_rng(seed)
    xyz = np.empty((n, 3))
    xyz[:, :2] = rng.uniform(-extent, extent, size=(n, 2))
    xyz[:, 2] = rng.uniform(-height, height, size=n)
    return xyz.astype(np.float32).astype(np.float64)


@pytest.mark.parametrize("n", [(1 << 20) + 17, MAX_POINTS])
def test_grid_select_many_tiles(orc, eng, n):
    xyz = _box_cloud(n, 40.0, 3.0, seed=n)
    for voxel in (0.1, 0.5):   # most points win / ~1 in 20 wins
        a = orc.grid_sample_indices(xyz, voxel)
        b = eng.grid_sample_indices(xyz, voxel)
        assert len(a) == len(b) and np.array_equal(a, b), voxel


def test_fused_sampler_many_tiles(orc, eng):
    xyz = _box_cloud(MAX_POINTS, 30.0, 3.0, seed=11)
    t = np.random.default_rng(12).uniform(0.0, 1.0, size=len(xyz))
    out = []
    for b in (orc, eng):
        o = _sequence_options(b, "GN", max_points_per_frame=MAX_POINTS)
        o.init_voxel_size = o.voxel_size = 0.2
        o.init_sample_voxel_size = o.sample_voxel_size = 3.0   # few keypoints: selection 2 still spans F positions
        od = b.odometry(o)
        s0 = od.RegisterFrame(xyz, t, 0)
        map0 = (od.MapSize(), od.GetMapPointer().export(0))
        s1 = od.RegisterFrame(xyz, t, 1)   # the first frame that samples keypoints
        assert s0.success and s1.success
        out.append((s0, map0, s1))
    (o0, (mo, (xo, vo)), o1), (e0, (me, (xe, ve)), e1) = out
    assert o0.num_corrected_points == e0.num_corrected_points
    assert mo == me and np.array_equal(vo, ve)
    assert np.abs(xo - xe).max() < POS_TOL
    assert o1.num_corrected_points > 1800 * 1024, o1.num_corrected_points   # > 1800 tiles in selection 2
    # (the selections run before the ICP; on a random box cloud the ICP itself is ill-posed, so poses are not compared)
    assert (o1.num_corrected_points, o1.num_keypoints) == (e1.num_corrected_points, e1.num_keypoints)
