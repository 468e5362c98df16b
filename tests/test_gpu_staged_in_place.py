"""A staged scan is read in place by RegisterStaged (no copy into the pipeline). Its summary point vectors must stay valid
after clear_staged() frees the staged scans (and other scans are staged into that memory), and a staged registration must
give the poses of the host-buffer path."""
import numpy as np
import pytest

import ct_icp_b200
from ct_icp_b200 import _abi as abi
from ct_icp_b200 import synthetic as syn


def _odometry(eng):
    o = eng.default_odometry_options()
    o.ct_icp_options.solver = abi.SOLVER["GN"]
    o.ct_icp_options.min_number_neighbors = 10
    o.map_options = eng.legacy_map_options(1.0, 20, 0.1)
    o.init_num_frames = 3
    o.debug_print = 0
    return eng.odometry(o)


def _pose(sm):
    return np.array(list(sm.frame.begin_pose.tr) + list(sm.frame.begin_pose.quat) + list(sm.frame.end_pose.tr) +
                    list(sm.frame.end_pose.quat))


@pytest.mark.gpu
def test_staged_scan_in_place_survives_clear_staged():
    eng = ct_icp_b200.engine()
    seq = syn.make_sequence(5, syn.SMALL16, seed=1234)
    od_host, od_staged = _odometry(eng), _odometry(eng)
    slots = [od_staged.stage_frame(s["xyz"], s["t"]) for s in seq]
    for i, s in enumerate(seq):
        a = od_host.RegisterFrame(s["xyz"], s["t"], s["frame_idx"])
        b = od_staged.RegisterStaged(slots[i], s["frame_idx"])
        assert a.success and b.success
        np.testing.assert_array_equal(_pose(a), _pose(b))
    kinds = (abi.POINTS_ALL_CORRECTED, abi.POINTS_CORRECTED, abi.POINTS_KEYPOINTS)
    before = [od_staged.points(w) for w in kinds]
    od_staged.clear_staged()
    # new scans of the same sizes are staged into memory the freed ones most likely occupied (cudaMalloc reuses it): a
    # pipeline still reading the freed scan would see their points
    for s in seq:
        od_staged.stage_frame(s["xyz"] * 2.0 + 100.0, s["t"])
    after = [od_staged.points(w) for w in kinds]
    for x, y in zip(before, after):
        assert x.tobytes() == y.tobytes()
    # the last scan of the host path is the same scan: its raw points and world points agree with the staged path's
    assert od_host.points(abi.POINTS_ALL_CORRECTED).tobytes() == after[0].tobytes()
    od_host.close()
    od_staged.close()
