"""Scoring trajectories on the device (cticp_kitti_evaluate, cticp_trajectory_kitti_evaluate, cticp_trajectory_metrics)
against the CPU restatement of kitti::EvaluatePoses and ComputeTrajectoryMetrics (tests/oracle_eval): exact pair and
segment selection, the distance arrays bit for bit, the scores within fp64 rounding, batches and repeated calls bit for
bit, the trajectory form against interpolate + evaluate, degenerate fits, refusals and short output capacities."""
import ctypes as C
import math

import numpy as np
import pytest

import ct_icp_b200
from ct_icp_b200 import _abi as abi
from conftest import get_sequence
from oracle_eval_lib import eval_oracle
from oracle_trajectory_lib import trajectory_oracle
from test_eval_oracle import _R, _line, _pose, _unit_quat, odometry_poses, perturbed, random_poses

pytestmark = pytest.mark.gpu

KITTI_FIELDS = ("mean_rpe", "mean_ape", "max_ape", "mean_local_err", "max_local_err")


@pytest.fixture(scope="module")
def eng():
    return ct_icp_b200.engine()


@pytest.fixture(scope="module")
def orc():
    return eval_oracle()


def _lengths(k):
    return ("driving", "indoor", (3.0, 25.0, 60.0, 250.0))[k % 3]


def _mean_close(a, b):
    """means: 1e-12 relative, or 1e-10 m absolute for the metre-valued ones near zero (ATE tolerance)"""
    if math.isnan(b):
        return math.isnan(a)
    return abs(a - b) <= max(1e-12 * abs(b), 1e-10)


def _check_kitti(r, o, lengths):
    lens = np.asarray(abi.KITTI_LENGTHS[lengths] if isinstance(lengths, str) else lengths)
    assert len(r["tab_errors"]) == len(o["tab_errors"])
    if len(o["tab_errors"]):
        np.testing.assert_allclose(r["tab_errors"][:, 0], o["tab_errors"][:, 0], rtol=0, atol=1e-11)
        # r_err within 3e-8 rad before the division by the length (acos near 1 amplifies rounding)
        d = np.abs(r["tab_errors"][:, 1] - o["tab_errors"][:, 1]) * lens.max()
        assert d.max() <= 3e-8, d.max()
    for k in KITTI_FIELDS:
        assert _mean_close(r[k], o[k]), (k, r[k], o[k])
    assert r["index_max_local_err"] == o["index_max_local_err"]


def _shape(rng, n, k):
    return odometry_poses(rng, n) if k % 2 == 0 else random_poses(rng, n)


@pytest.mark.parametrize("n", [1, 2, 6, 7, 10, 11, 1000, 4541])
@pytest.mark.parametrize("B", [1, 3, 16])
def test_kitti_against_the_oracle(eng, orc, n, B):
    rng = np.random.default_rng(n * 100 + B)
    for k in range(3):
        gt = _shape(rng, n, k)
        ests = [perturbed(rng, gt) for _ in range(B)]
        lengths = _lengths(k)
        r = eng.kitti_evaluate(gt, ests, lengths)
        o = orc.kitti_evaluate(gt, ests, lengths)
        for rb, ob in zip(r, o):
            _check_kitti(rb, ob, lengths)
        assert eng.trajectory_distances(gt, "kitti").tobytes() == orc.trajectory_distances(gt, "kitti").tobytes()
        assert eng.trajectory_distances(gt, "metrics").tobytes() == orc.trajectory_distances(gt, "metrics").tobytes()


def _sv(ref, tgt):
    M = (tgt - tgt.mean(axis=0)).T @ (ref - ref.mean(axis=0))
    return np.linalg.svd(M, compute_uv=False)


def _separated(s):
    return s[2] > 1e-6 * s[0] and (s[0] - s[1]) > 1e-6 * s[0] and (s[1] - s[2]) > 1e-6 * s[0]


def _rot_tol(s):
    """1e-12, widened by the fit's conditioning: a rounding of M moves the rotation by about eps s0 / (smallest gap)"""
    return max(1e-12, 4e-15 * s[0] / min(s[2], s[0] - s[1], s[1] - s[2]))


def _check_metrics(r, o, gt, est):
    assert r["num_segments"] == o["num_segments"]
    assert r["total_distance"] == o["total_distance"]
    rs, os_ = r["segments"], o["segments"]
    assert np.array_equal(rs["start_idx"], os_["start_idx"]) and np.array_equal(rs["end_idx"], os_["end_idx"])
    assert rs["segment_length"].tobytes() == os_["segment_length"].tobytes()
    np.testing.assert_allclose(rs["loc_error"], os_["loc_error"], rtol=0, atol=1e-10)
    assert abs(r["mean_ate"] - o["mean_ate"]) <= 1e-10 and abs(r["max_ate"] - o["max_ate"]) <= 1e-10
    assert r["max_ate_idx"] == o["max_ate_idx"]
    for k in ("segment_mean_ate", "segment_mean_ate_ratio"):
        assert _mean_close(r[k], o[k]), (k, r[k], o[k])
    ref = np.array([p.tr[:] for p in gt])
    tgt = np.array([p.tr[:] for p in est])
    sv = _sv(ref, tgt)
    if _separated(sv):
        np.testing.assert_allclose(r["quat"], o["quat"], rtol=0, atol=_rot_tol(sv))
        np.testing.assert_allclose(r["tr"], o["tr"], rtol=0, atol=_rot_tol(sv) * (1.0 + np.abs(ref).max()))
    for a, b in zip(rs, os_):
        s, e = int(a["start_idx"]), int(a["end_idx"]) + 1
        sv = _sv(ref[s:e], tgt[s:e])
        if _separated(sv):
            np.testing.assert_allclose(a["quat"], b["quat"], rtol=0, atol=_rot_tol(sv))


@pytest.mark.parametrize("n", [6, 7, 10, 11, 1000, 4541])
@pytest.mark.parametrize("B", [1, 3, 16])
def test_metrics_against_the_oracle(eng, orc, n, B):
    rng = np.random.default_rng(n * 10 + B)
    for k in range(2):
        gt = _shape(rng, n, k)
        ests = [perturbed(rng, gt) for _ in range(B)]
        seg_len = 10.0 if k == 0 else 150.0
        r = eng.trajectory_metrics(gt, ests, seg_len)
        o = orc.trajectory_metrics(gt, ests, seg_len)
        for rb, ob, e in zip(r, o, ests):
            _check_metrics(rb, ob, gt, e)


def _bytes(d):
    return b"".join(np.asarray(v).tobytes() for _, v in sorted(d.items()))


def test_batches_and_repeated_calls_are_bit_identical(eng):
    rng = np.random.default_rng(77)
    gt = odometry_poses(rng, 2000)
    ests = [perturbed(rng, gt) for _ in range(16)]
    kb = eng.kitti_evaluate(gt, ests, "driving")
    mb = eng.trajectory_metrics(gt, ests, 10.0)
    for b in (0, 5, 15):
        assert _bytes(eng.kitti_evaluate(gt, ests[b], "driving")) == _bytes(kb[b])
        assert _bytes(eng.trajectory_metrics(gt, ests[b], 10.0)) == _bytes(mb[b])
    assert [_bytes(x) for x in eng.kitti_evaluate(gt, ests, "driving")] == [_bytes(x) for x in kb]
    assert [_bytes(x) for x in eng.trajectory_metrics(gt, ests, 10.0)] == [_bytes(x) for x in mb]


def test_trajectory_form_equals_interpolate_then_evaluate(eng, orc):
    rng = np.random.default_rng(31)
    gt = odometry_poses(rng, 1200)
    est = perturbed(rng, gt)
    frames = []
    for i in range(0, len(est) - 1, 2):   # begin / end poses of frames, timestamps shifted off the ground truth's
        f = abi.Frame()
        f.begin_pose, f.end_pose = est[i], est[i + 1]
        f.begin_pose.dest_timestamp += 0.03
        f.end_pose.dest_timestamp += 0.03
        f.begin_pose.dest_frame_id = f.end_pose.dest_frame_id = i // 2
        frames.append(f)
    traj = eng.continuous_trajectory(frames)
    ts = np.array([p.dest_timestamp for p in gt])
    for lengths in ("driving", "indoor"):
        r = traj.kitti_evaluate(gt, lengths)
        interp = traj.interpolate(ts)
        assert _bytes(r) == _bytes(eng.kitti_evaluate(gt, interp, lengths))
        otraj = trajectory_oracle().continuous_trajectory(frames)
        _check_kitti(r, orc.kitti_evaluate(gt, otraj.interpolate(ts), lengths), lengths)


def test_a_registered_sequence_scored_at_mid_frame(eng, orc):
    seq = get_sequence("small16", 8)
    o = eng.default_odometry_options()
    o.ct_icp_options.solver = abi.SOLVER["GN"]
    o.ct_icp_options.min_number_neighbors = 10
    o.map_options = eng.legacy_map_options(1.0, 20, 0.1)
    o.init_num_frames = 3
    o.debug_print = 0
    o.ct_icp_options.debug_print = 0
    od = eng.odometry(o)
    for s in seq:
        assert od.RegisterFrame(s["xyz"], s["t"], s["frame_idx"]).success
    T0inv = np.linalg.inv(seq[0]["gt_begin"])
    gt = []
    for s in seq:   # the ground-truth mid-frame pose (the regression runner's comparison), relative to the first pose
        Tb, Te = T0inv @ s["gt_begin"], T0inv @ s["gt_end"]
        from scipy.spatial.transform import Rotation, Slerp
        q = Slerp([0, 1], Rotation.from_matrix([Tb[:3, :3], Te[:3, :3]]))([0.5]).as_quat()[0]
        gt.append(_pose(q, 0.5 * (Tb[:3, 3] + Te[:3, 3]), 0.5 * (s["t"].min() + s["t"].max()), s["frame_idx"]))
    traj = eng.continuous_trajectory(od.Trajectory())
    otraj = trajectory_oracle().continuous_trajectory(od.Trajectory())
    ts = np.array([p.dest_timestamp for p in gt])
    r = traj.kitti_evaluate(gt, (0.5, 1.0))
    _check_kitti(r, orc.kitti_evaluate(gt, otraj.interpolate(ts), (0.5, 1.0)), (0.5, 1.0))
    assert r["mean_ape"] < 0.5
    est = traj.interpolate(ts)
    _check_metrics(eng.trajectory_metrics(gt, est, 0.5), orc.trajectory_metrics(gt, est, 0.5), gt,
                   [_pose(p["quat"], p["tr"]) for p in est])


def test_rigid_transform_scores_zero_and_identical_estimates_score_zero(eng):
    rng = np.random.default_rng(1234)
    gt = [_pose(_unit_quat(rng), rng.uniform(-1, 1, 3) * 100, i, i) for i in range(1000)]
    q, t = _unit_quat(rng), rng.uniform(-1, 1, 3)
    R = _R(q)
    est = []
    for p in gt:
        qb = np.array(p.quat[:])
        w = q[3] * qb[3] - q[:3] @ qb[:3]
        v = q[3] * qb[:3] + qb[3] * q[:3] + np.cross(q[:3], qb[:3])
        qq = np.append(v, w)
        est.append(_pose(qq / np.linalg.norm(qq), R @ np.array(p.tr[:]) + t, p.dest_timestamp, p.dest_frame_id))
    m = eng.trajectory_metrics(gt, est, 1000.0)
    for k in ("max_ate", "mean_ate", "segment_mean_ate", "segment_mean_ate_ratio"):
        assert m[k] <= 1e-12, (k, m[k])
    gt = odometry_poses(rng, 3000)
    k = eng.kitti_evaluate(gt, gt, (100.0,))
    assert k["mean_ape"] <= 1e-10 and k["max_local_err"] == 0.0 and k["index_max_local_err"] == 0
    assert np.abs(k["tab_errors"][:, 0]).max() <= 1e-11 and k["mean_rpe"] <= 1e-9
    assert np.abs(k["tab_errors"][:, 1] * 100.0).max() <= 3e-8   # acos near 1: ~1e-8 rad rather than 0
    m = eng.trajectory_metrics(gt, gt, 10.0)
    assert m["max_ate"] <= 1e-10 and m["segment_mean_ate"] <= 1e-10


def test_degenerate_fits_match_the_oracle(eng, orc):
    gt = _line(40, 0.7)
    still = [_pose((0, 0, 0, 1), (5.0, -2.0, 1.0), i, i) for i in range(40)]    # stationary: M = 0
    straight = [_pose((0, 0, 0, 1), (0.0, 0.7 * i, 3.0), i, i) for i in range(40)]   # both straight: rank 1
    rng = np.random.default_rng(3)
    noisy = perturbed(rng, gt, 0.0, 0.05)                                          # straight ground truth only
    for est in (still, straight, noisy):
        r = eng.trajectory_metrics(gt, est, 4.0)
        o = orc.trajectory_metrics(gt, est, 4.0)
        for k in ("mean_ate", "max_ate", "segment_mean_ate", "segment_mean_ate_ratio"):
            assert np.isfinite(r[k]) and abs(r[k] - o[k]) <= 1e-10, (k, r[k], o[k])
        np.testing.assert_allclose(r["segments"]["loc_error"], o["segments"]["loc_error"], rtol=0, atol=1e-10)
        assert np.isfinite(r["quat"]).all() and np.isfinite(r["segments"]["quat"]).all()
    r = eng.trajectory_metrics(gt, still, 4.0)
    assert np.array_equal(r["quat"], [0, 0, 0, 1]) and (r["segments"]["quat"] == [0, 0, 0, 1]).all()


def _c_poses(poses):
    arr = np.zeros(len(poses), dtype=abi.pose_dtype())
    for i, p in enumerate(poses):
        C.memmove(arr.ctypes.data + i * arr.itemsize, C.addressof(p), C.sizeof(abi.Pose))
    return arr


def test_refusals_leave_outputs_untouched(eng):
    rng = np.random.default_rng(8)
    gt = _c_poses(odometry_poses(rng, 50))
    est = _c_poses(perturbed(rng, odometry_poses(rng, 50)))
    lens = np.array([5.0, 10.0])
    kf, mf = eng.fn("kitti_evaluate"), eng.fn("trajectory_metrics")

    def kitti(g=gt, n=None, e=est, B=1, ln=lens, nl=None, out=True):
        o = (abi.KittiErrors * 2)()
        C.memset(o, 0x5A, C.sizeof(o))
        tab = np.full((2, 64, 2), 7.0)
        rc = kf(0, g.ctypes.data if g is not None else None, len(gt) if n is None else n,
                e.ctypes.data if e is not None else None, B, ln.ctypes.data if ln is not None else None,
                (len(ln) if ln is not None else 0) if nl is None else nl, o if out else None, tab.ctypes.data, 64)
        assert rc == abi.ERR_INVALID_ARGUMENT, rc
        assert bytes(o) == b"\x5a" * C.sizeof(o) and (tab == 7.0).all()

    def metrics(g=gt, n=None, e=est, B=1, seg=10.0, out=True):
        o = (abi.TrajMetrics * 2)()
        C.memset(o, 0x5A, C.sizeof(o))
        segs = np.full(2 * 64 * C.sizeof(abi.TrajSegment), 0x33, dtype=np.uint8)
        rc = mf(0, g.ctypes.data if g is not None else None, len(gt) if n is None else n,
                e.ctypes.data if e is not None else None, B, seg, o if out else None, segs.ctypes.data, 64)
        assert rc == abi.ERR_INVALID_ARGUMENT, rc
        assert bytes(o) == b"\x5a" * C.sizeof(o) and (segs == 0x33).all()

    kitti(n=0)
    kitti(B=0)
    kitti(g=None)
    kitti(e=None)
    kitti(out=False)
    kitti(ln=None)
    kitti(nl=0)
    for bad in (0.0, -1.0, np.nan, np.inf):
        kitti(ln=np.array([10.0, bad]))
    metrics(n=0)
    metrics(n=5)
    metrics(B=0)
    metrics(g=None)
    metrics(e=None)
    metrics(out=False)
    for bad in (0.0, -3.0, np.nan, np.inf):
        metrics(seg=bad)
    for field, k, bad in (("quat", None, 0.0), ("quat", 2, np.nan), ("tr", 1, np.inf), ("dest_timestamp", None, np.nan)):
        for which in ("gt", "est"):
            if field == "dest_timestamp" and which == "est":
                continue
            g, e = gt.copy(), est.copy()
            a = g if which == "gt" else e
            if k is None:
                a[field][17] = bad
            else:
                a[field][17, k] = bad
            kitti(g=g, e=e)
            metrics(g=g, e=e)
    with pytest.raises(ct_icp_b200._binding.CticpError):   # an estimate whose count differs from the ground truth's
        eng.kitti_evaluate(odometry_poses(rng, 50), [odometry_poses(rng, 49)])
    traj = eng.continuous_trajectory(odometry_poses(rng, 50))
    o = abi.KittiErrors()
    rc = eng.fn("trajectory_kitti_evaluate")(traj.h, gt.ctypes.data, len(gt), None, 0, C.byref(o), None, 0)
    assert rc == abi.ERR_INVALID_ARGUMENT


def test_short_capacity_writes_min_cap_count(eng):
    rng = np.random.default_rng(12)
    gt = _c_poses(odometry_poses(rng, 800))
    est = np.concatenate([_c_poses(perturbed(rng, odometry_poses(rng, 800))) for _ in range(2)])
    lens = np.array([10.0, 50.0])
    out = (abi.KittiErrors * 2)()
    full = np.zeros((2, 400, 2))
    count = eng.fn("kitti_evaluate")(0, gt.ctypes.data, 800, est.ctypes.data, 2, lens.ctypes.data, 2, out,
                                     full.ctypes.data, 400)
    assert 5 < count <= 160
    short = np.full((2, 5, 2), -1.0)
    assert eng.fn("kitti_evaluate")(0, gt.ctypes.data, 800, est.ctypes.data, 2, lens.ctypes.data, 2, out,
                                    short.ctypes.data, 5) == count
    assert short.tobytes() == full[:, :5].tobytes()
    mo = (abi.TrajMetrics * 2)()
    segs = np.zeros((2, 200), dtype=abi.traj_segment_dtype())
    sc = eng.fn("trajectory_metrics")(0, gt.ctypes.data, 800, est.ctypes.data, 2, 10.0, mo, segs.ctypes.data, 200)
    assert sc > 3
    few = np.full((2, 3), 0, dtype=abi.traj_segment_dtype())
    few["loc_error"] = -1.0
    assert eng.fn("trajectory_metrics")(0, gt.ctypes.data, 800, est.ctypes.data, 2, 10.0, mo, few.ctypes.data, 3) == sc
    assert few.tobytes() == segs[:, :3].tobytes()
