"""CPU tests of the restatement of slam::LinearContinuousTrajectory (tests/oracle_trajectory) that the GPU tests of the
continuous trajectory compare the engine against: the reference's own unit cases (test/unit/SlamCore/test_trajectory.cxx)
as seeded fixtures, its quirks, and its consistency checks."""
import ctypes as C
import math

import numpy as np
import pytest

import ct_icp_b200
from ct_icp_b200 import _abi as abi
from oracle_trajectory_lib import trajectory_oracle


@pytest.fixture(scope="module")
def tor():
    b = trajectory_oracle()
    f = b.fn("trajectory_closest_ids")
    f.restype = C.c_int
    f.argtypes = [C.c_void_p, C.c_double, C.c_int64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    return b


def closest(b, traj, t, frame_id=None):
    lo, up = C.c_uint64(), C.c_uint64()
    b.check(b.fn("trajectory_closest_ids")(traj.h, t, -1 if frame_id is None else frame_id, C.byref(lo), C.byref(up)))
    return lo.value, up.value


def pose(quat, tr, ts, fid, ref_fid=0, ref_ts=0.0):
    p = abi.Pose.make(quat=quat, tr=tr, dest_timestamp=ts, dest_frame_id=fid)
    p.ref_frame_id, p.ref_timestamp = ref_fid, ref_ts
    return p


def unit_random_quat(rng):
    q = rng.normal(size=4)
    return q / np.linalg.norm(q)


def eigen_slerp(a, b, t):
    """Eigen QuaternionBase::slerp in fp64 (not renormalised)"""
    one = 1.0 - np.finfo(np.float64).eps
    d = float(np.dot(a, b))
    ad = abs(d)
    if ad >= one:
        s0, s1 = 1.0 - t, t
    else:
        th = math.acos(ad)
        s0, s1 = math.sin((1.0 - t) * th) / math.sin(th), math.sin(t * th) / math.sin(th)
    if d < 0:
        s1 = -s1
    return s0 * np.asarray(a) + s1 * np.asarray(b)


def eight_poses(seed=7):
    """test_definition: 8 poses over 4 frames, random unit quaternions and translations in [-1, 1]"""
    rng = np.random.default_rng(seed)
    spec = [(0.0, 0), (0.5, 0), (0.9, 0), (1.01, 1), (1.3, 1), (1.5, 1), (2.0, 2), (3.0, 3)]
    return [pose(unit_random_quat(rng), rng.uniform(-1, 1, 3), ts, fid) for ts, fid in spec]


def test_reference_definition_case(tor):
    poses = eight_poses()
    traj = tor.continuous_trajectory(poses[::-1])   # Create sorts
    got = traj.poses()
    assert list(got["dest_timestamp"]) == [0.0, 0.5, 0.9, 1.01, 1.3, 1.5, 2.0, 3.0]
    assert min(got["dest_timestamp"]) == 0.0 and max(got["dest_timestamp"]) == 3.0
    p_min = traj.interpolate([0.0])[0]
    assert list(p_min["quat"]) == list(poses[0].quat) and list(p_min["tr"]) == list(poses[0].tr)
    # InterpolatePose(1.0): poses 2 (0.9) and 3 (1.01); InterpolatePoseWithFrameId(1.1, 1): poses 3 (1.01) and 4 (1.3)
    for t, fid, (i, j) in ((1.0, None, (2, 3)), (1.1, 1, (3, 4))):
        p = traj.interpolate([t], None if fid is None else [fid])[0]
        a, b = poses[i], poses[j]
        alpha = (t - a.dest_timestamp) / (b.dest_timestamp - a.dest_timestamp)
        assert np.all(np.isfinite(p["quat"])) and np.all(np.isfinite(p["tr"]))
        np.testing.assert_allclose(p["quat"], eigen_slerp(list(a.quat), list(b.quat), alpha), rtol=0, atol=1e-15)
        np.testing.assert_allclose(p["tr"], (1 - alpha) * np.array(a.tr) + alpha * np.array(b.tr), rtol=0, atol=1e-15)
        assert p["dest_timestamp"] == pytest.approx(t, abs=1e-15)
        assert p["dest_frame_id"] == a.dest_frame_id and p["ref_frame_id"] == a.ref_frame_id


def test_reference_closest_pose_tables(tor):
    rng = np.random.default_rng(11)
    four = tor.continuous_trajectory([pose(unit_random_quat(rng), rng.uniform(-1, 1, 3), float(k), k) for k in range(4)])
    assert closest(tor, four, 0.0) == (0, 0)
    assert closest(tor, four, 0.0, 0) == (0, 0)
    assert closest(tor, four, 0.5, 0) == (0, 1)
    assert closest(tor, four, 1.0, 0) == (0, 1)
    assert closest(tor, four, 1.0, 1) == (0, 1)
    # FindClosestPose (:102-126; clip_on_bounds only matters where the bounds check fires, which none of these reach)
    three = tor.continuous_trajectory([pose((0, 0, 0, 1), (0, 0, 0), float(k), k) for k in range(3)])
    for (t, fid), ids in (((1.0, 1), (0, 1)), ((2.0, 2), (1, 2)), ((1.5, 2), (1, 2)), ((1.5, 1), (1, 2)),
                          ((1.0, 0), (0, 1))):
        assert closest(tor, three, t, fid) == ids, (t, fid)


def odometry_shaped(rng, n_frames, equal_boundaries):
    frames = []
    t = 10.0
    for k in range(n_frames):
        b = t
        e = b + 0.1
        t = e if equal_boundaries else e + 0.01
        f = abi.Frame()
        f.begin_pose = pose(unit_random_quat(rng), rng.uniform(-5, 5, 3), b, k)
        f.end_pose = pose(unit_random_quat(rng), rng.uniform(-5, 5, 3), e, k)
        frames.append(f)
    return frames


def test_alpha_quirks(tor):
    rng = np.random.default_rng(3)
    frames = odometry_shaped(rng, 3, equal_boundaries=True)
    traj = tor.continuous_trajectory(frames)
    P = traj.poses()
    # above the pair → alpha 0: frame 0 queried past its end pairs its end pose with frame 1's begin pose
    t = float(P[1]["dest_timestamp"]) + 0.05
    p = traj.interpolate([t], [0])[0]
    assert closest(tor, traj, t, 0) == (1, 2)
    assert p["dest_timestamp"] == P[1]["dest_timestamp"] and list(p["tr"]) == list(P[1]["tr"])
    # equal timestamps → alpha 1: frame 1 at its begin timestamp pairs frame 0's end (same timestamp) with its begin
    t = float(P[2]["dest_timestamp"])
    assert P[1]["dest_timestamp"] == t
    p = traj.interpolate([t], [1])[0]
    assert closest(tor, traj, t, 1) == (1, 2)
    assert list(p["tr"]) == list(P[2]["tr"]) and p["dest_timestamp"] == t
    assert p["dest_frame_id"] == 0                              # from the lower pose
    # NaN → pose 0, unchanged
    p = traj.interpolate([float("nan")])[0]
    assert p.tobytes() == P[0].tobytes()
    # below the minimum → pose 0, above the maximum → the last pose, both unchanged
    assert traj.interpolate([-100.0])[0].tobytes() == P[0].tobytes()
    assert traj.interpolate([1e9])[0].tobytes() == P[-1].tobytes()


def test_bounds_check_as_written(tor):
    """Min >= t && t >= Max only holds when every timestamp is the same positive value: then such a t takes pose 0,
    whatever the frame id"""
    traj = tor.continuous_trajectory([pose((0, 0, 0, 1), (1, 0, 0), 2.0, 0), pose((0, 0, 0, 1), (2, 0, 0), 2.0, 1)])
    assert closest(tor, traj, 2.0, 1) == (0, 0)
    assert closest(tor, traj, 2.0) == (0, 0)
    assert traj.interpolate([2.0], [1])[0]["tr"][0] == 1.0
    assert traj.interpolate([2.0], [7])[0]["tr"][0] == 1.0       # a frame beyond, but clipped before the CHECK
    # MaxTimestamp starts at DBL_MIN: with timestamps <= 0 the check never fires
    neg = tor.continuous_trajectory([pose((0, 0, 0, 1), (1, 0, 0), -1.0, 0), pose((0, 0, 0, 1), (2, 0, 0), -1.0, 1)])
    assert closest(tor, neg, -1.0, 1) == (0, 1)


def test_frame_ids_absent_and_beyond(tor):
    traj = tor.continuous_trajectory([pose((0, 0, 0, 1), (float(k), 0, 0), float(k), 2 * k) for k in range(3)])
    assert closest(tor, traj, 1.5, 1) == (0, 1)         # frame 1 is absent: the pair around where it would sort
    assert closest(tor, traj, 0.5, 3) == (1, 2)
    assert closest(tor, traj, 9.0, 4) == (2, 2)         # the last frame, past its last pose
    with pytest.raises(ct_icp_b200.CticpError) as e:
        traj.interpolate([1.0], [5])
    assert e.value.code == abi.ERR_INVALID_ARGUMENT


@pytest.mark.parametrize("case", ["empty", "reference_frame", "decreasing", "nan"])
def test_consistency_errors(tor, case):
    ok = [pose((0, 0, 0, 1), (0, 0, 0), 0.0, 0), pose((0, 0, 0, 1), (0, 0, 0), 1.0, 1)]
    if case == "empty":
        poses = []
    elif case == "reference_frame":
        poses = ok + [pose((0, 0, 0, 1), (0, 0, 0), 2.0, 2, ref_fid=3)]
    elif case == "decreasing":
        poses = ok + [pose((0, 0, 0, 1), (0, 0, 0), 0.5, 2)]
    else:
        poses = ok + [pose((0, 0, 0, 1), (0, 0, 0), float("nan"), 2)]
    with pytest.raises(ct_icp_b200.CticpError) as e:
        tor.continuous_trajectory(poses)
    assert e.value.code == abi.ERR_INVALID_ARGUMENT
    # within one frame the order of timestamps is free: Create sorts them
    tor.continuous_trajectory(ok + [pose((0, 0, 0, 1), (0, 0, 0), 1.5, 1), pose((0, 0, 0, 1), (0, 0, 0), 1.2, 1)])


def test_equal_keys_keep_their_order(tor):
    poses = [pose((0, 0, 0, 1), (float(k), 0, 0), 1.0, 0) for k in range(5)] + [pose((0, 0, 0, 1), (9, 0, 0), 0.0, 0)]
    got = tor.continuous_trajectory(poses).poses()
    assert list(got["tr"][:, 0]) == [9.0, 0.0, 1.0, 2.0, 3.0, 4.0]


def test_transform_is_interpolate_then_apply(tor):
    rng = np.random.default_rng(5)
    frames = odometry_shaped(rng, 4, equal_boundaries=False)
    traj = tor.continuous_trajectory(frames)
    n = 200
    xyz = rng.uniform(-50, 50, (n, 3))
    t = rng.uniform(9.9, 10.5, n)
    w = traj.transform(xyz, t)
    P = traj.interpolate(t)
    for i in range(n):
        q = P[i]["quat"] / math.sqrt(float(np.dot(P[i]["quat"], P[i]["quat"])))
        v, s = q[:3], q[3]
        uv = 2 * np.cross(v, xyz[i])
        np.testing.assert_allclose(w[i], xyz[i] + s * uv + np.cross(v, uv) + P[i]["tr"], rtol=0, atol=1e-12)
    # segments select the frame-id lookup
    ends = np.array([50, 120, 200])
    fids = np.array([0, 2, 3])
    w2 = traj.transform(xyz, t, segments=(ends, fids))
    P2 = traj.interpolate(t, np.repeat(fids, np.diff(np.concatenate([[0], ends]))))
    for i in range(0, n, 17):
        q = P2[i]["quat"] / np.linalg.norm(P2[i]["quat"])
        v, s = q[:3], q[3]
        uv = 2 * np.cross(v, xyz[i])
        np.testing.assert_allclose(w2[i], xyz[i] + s * uv + np.cross(v, uv) + P2[i]["tr"], rtol=0, atol=1e-12)


def test_engine_without_device_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(ct_icp_b200.CticpError) as e:
        ct_icp_b200.engine().continuous_trajectory([pose((0, 0, 0, 1), (0, 0, 0), 0.0, 0)])
    assert e.value.code == abi.ERR_NO_DEVICE
