"""The CPU restatement of kitti::EvaluatePoses and ComputeTrajectoryMetrics (tests/oracle_eval) against an independent
NumPy restatement, the reference's quirks on hand-built cases, the reference's own unit test (test/unit/SlamCore/
test_eval.cxx: a rigid transform of the ground truth scores zero), and the ctypes layouts of the new C structs."""
import ctypes as C
import math

import numpy as np
import pytest

from ct_icp_b200 import _abi as abi
from oracle_eval_lib import eval_oracle


@pytest.fixture(scope="module")
def orc():
    return eval_oracle()


def _pose(quat, tr, ts=0.0, fid=0):
    return abi.Pose.make(quat=tuple(float(v) for v in quat), tr=tuple(float(v) for v in tr), dest_timestamp=float(ts),
                         dest_frame_id=fid)


def _unit_quat(rng):
    q = rng.normal(size=4)
    return q / np.linalg.norm(q)


def random_poses(rng, n):
    return [_pose(_unit_quat(rng), rng.uniform(-100, 100, 3), i, i) for i in range(n)]


def odometry_poses(rng, n, step=0.8):
    """a vehicle-like path: heading drifts slowly, ~step m per pose, small roll / pitch noise"""
    poses, yaw, tr = [], 0.0, np.zeros(3)
    for i in range(n):
        yaw += rng.normal(scale=0.02)
        q = np.array([rng.normal(scale=0.005), rng.normal(scale=0.005), math.sin(yaw / 2), math.cos(yaw / 2)])
        q /= np.linalg.norm(q)
        poses.append(_pose(q, tr, 0.1 * i, i))
        tr = tr + step * np.array([math.cos(yaw), math.sin(yaw), 0.01 * rng.normal()])
    return poses


def perturbed(rng, poses, rot=0.01, tr=0.3):
    out = []
    for p in poses:
        q = np.array(p.quat[:]) + rng.normal(scale=rot, size=4)
        out.append(_pose(q / np.linalg.norm(q), np.array(p.tr[:]) + rng.normal(scale=tr, size=3), p.dest_timestamp,
                         p.dest_frame_id))
    return out


# ---- the NumPy restatement ---------------------------------------------------------------------------------------------
def _R(q):
    x, y, z, w = np.asarray(q) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _M(p):
    m = np.eye(4)
    m[:3, :3] = _R(p.quat[:])
    m[:3, 3] = p.tr[:]
    return m


def _n3(x, y, z):   # sqrt((x*x + y*y) + z*z): the oracle's roundings, so the pair and segment choices agree exactly
    return math.sqrt(x * x + y * y + z * z)


def np_kitti(gt, est, lengths):
    n = len(gt)
    G, E = [_M(p) for p in gt], [_M(p) for p in est]
    ape = [np.linalg.norm((np.linalg.inv(E[i]) @ G[i])[:3, 3]) for i in range(n)]
    loc = [abs(np.linalg.norm(G[i][:3, 3] - G[i - 1][:3, 3]) - np.linalg.norm(E[i][:3, 3] - E[i - 1][:3, 3]))
           for i in range(1, n)]
    dist = [0.0]
    for i in range(1, n):
        a, b = gt[i - 1].tr, gt[i].tr
        dist.append(dist[-1] + _n3(a[0] - b[0], a[1] - b[1], a[2] - b[2]))
    pairs, tab = [], []
    for first in range(0, n, 10):
        for ln in lengths:
            last = next((i for i in range(first, n) if dist[i] > dist[first] + ln), None)
            if last is None:
                continue
            err = np.linalg.inv(np.linalg.inv(E[first]) @ E[last]) @ (np.linalg.inv(G[first]) @ G[last])
            d = 0.5 * (np.trace(err[:3, :3]) - 1.0)
            tab.append((np.linalg.norm(err[:3, 3]) / ln, math.acos(max(min(d, 1.0), -1.0)) / ln))
            pairs.append((first, last))
    with np.errstate(invalid="ignore", divide="ignore"):
        mean_rpe = np.float64(sum(t for t, _ in tab)) / np.float64(len(tab)) * 100.0
        mean_loc = np.float64(sum(loc)) / np.float64(n - 1)
    mx_loc = max(loc) if loc else 0.0
    idx = 1 + loc.index(mx_loc) if loc and mx_loc > 0 else 0
    return dict(mean_rpe=mean_rpe, mean_ape=sum(ape) / n, max_ape=max(ape), mean_local_err=mean_loc,
                max_local_err=mx_loc, index_max_local_err=idx, tab_errors=np.array(tab).reshape(-1, 2), pairs=pairs)


def np_procrustes(ref, tgt):
    cr, ct = ref.mean(axis=0), tgt.mean(axis=0)
    M = (tgt - ct).T @ (ref - cr)
    U, _, Vt = np.linalg.svd(M)
    R = U @ Vt
    if np.linalg.det(R) < 0:
        R = U @ np.diag([1.0, 1.0, -1.0]) @ Vt
    return R, ct - R @ cr


def _se3_inv_tr_norm(a, b):
    """|(a.Inverse() * b).tr| in TSE3 arithmetic, written out with the oracle's roundings"""
    def qrot(q, v):
        x, y, z, w = q
        uv = (y * v[2] - z * v[1], z * v[0] - x * v[2], x * v[1] - y * v[0])
        uv = tuple(u + u for u in uv)
        c = (y * uv[2] - z * uv[1], z * uv[0] - x * uv[2], x * uv[1] - y * uv[0])
        return tuple(v[k] + w * uv[k] + c[k] for k in range(3))
    x, y, z, w = a.quat[:]
    n2 = x * x + y * y + z * z + w * w
    qi = (-x / n2, -y / n2, -z / n2, w / n2)
    ti = qrot(qi, a.tr[:])
    ni = math.sqrt(qi[0] * qi[0] + qi[1] * qi[1] + qi[2] * qi[2] + qi[3] * qi[3])
    r = qrot(tuple(c / ni for c in qi), b.tr[:])
    return _n3(r[0] + -ti[0], r[1] + -ti[1], r[2] + -ti[2])


def np_metrics(gt, est, seg_len):
    n = len(gt)
    ref = np.array([p.tr[:] for p in gt])
    tgt = np.array([p.tr[:] for p in est])
    dist = [0.0]
    for i in range(n - 1):
        dist.append(dist[-1] + _se3_inv_tr_norm(gt[i], gt[i + 1]))
    R, t = np_procrustes(ref, tgt)
    ate = np.linalg.norm(ref @ R.T + t - tgt, axis=1)
    max_idx = -1
    mx = 0.0
    for i, a in enumerate(ate):
        if a > mx:
            mx, max_idx = a, i
    segs, start, last = [], 0, 0.0
    for idx in range(n):
        if dist[idx] - last > seg_len:
            if idx - start + 1 > 5:
                Rs, ts = np_procrustes(ref[start:idx + 1], tgt[start:idx + 1])
                loc = np.linalg.norm(ref[start:idx + 1] @ Rs.T + ts - tgt[start:idx + 1], axis=1).max()
                segs.append((start, idx, dist[idx] - last, loc))
            start, last = idx, dist[idx]
    with np.errstate(invalid="ignore", divide="ignore"):
        sm = np.float64(sum(s[3] for s in segs)) / np.float64(len(segs))
        sr = np.float64(sum(s[3] / s[2] for s in segs)) / np.float64(len(segs))
    return dict(total_distance=dist[-1], dist=np.array(dist), mean_ate=ate.mean(), max_ate=mx, max_ate_idx=max_idx,
                segments=segs, segment_mean_ate=sm, segment_mean_ate_ratio=sr)


def _close(a, b, tol):
    return (math.isnan(a) and math.isnan(b)) or abs(a - b) <= tol


CASES = [(n, shape) for n in (1, 2, 6, 7, 11, 1000) for shape in ("random", "odometry")]


@pytest.mark.parametrize("n,shape", CASES)
def test_kitti_oracle_against_numpy(orc, n, shape):
    rng = np.random.default_rng(1000 + n)
    gt = random_poses(rng, n) if shape == "random" else odometry_poses(rng, n)
    est = perturbed(rng, gt)
    lengths = (50.0, 100.0, 150.0) if shape == "random" else (5.0, 10.0, 40.0, 100.0)
    r = orc.kitti_evaluate(gt, est, lengths)
    ref = np_kitti(gt, est, lengths)
    assert len(r["tab_errors"]) == len(ref["tab_errors"])
    np.testing.assert_allclose(r["tab_errors"][:, 0], ref["tab_errors"][:, 0], rtol=0, atol=1e-11)
    np.testing.assert_allclose(r["tab_errors"][:, 1], ref["tab_errors"][:, 1], rtol=0, atol=3e-8)
    for k in ("mean_rpe", "mean_ape", "max_ape", "mean_local_err", "max_local_err"):
        assert _close(r[k], ref[k], 1e-9 * max(1.0, abs(ref[k]) if not math.isnan(ref[k]) else 1.0)), (k, r[k], ref[k])
    assert r["index_max_local_err"] == ref["index_max_local_err"]
    d = orc.trajectory_distances(gt, "kitti")
    assert len(d) == n and d[0] == 0.0


@pytest.mark.parametrize("n,shape", [c for c in CASES if c[0] >= 6])
def test_metrics_oracle_against_numpy(orc, n, shape):
    rng = np.random.default_rng(2000 + n)
    gt = random_poses(rng, n) if shape == "random" else odometry_poses(rng, n)
    est = perturbed(rng, gt)
    seg_len = 150.0 if shape == "random" else 10.0
    r = orc.trajectory_metrics(gt, est, seg_len)
    ref = np_metrics(gt, est, seg_len)
    assert np.array_equal(orc.trajectory_distances(gt, "metrics"), ref["dist"])   # bit for bit
    assert r["total_distance"] == ref["total_distance"]
    assert r["num_segments"] == len(ref["segments"])
    segs = r["segments"]
    assert [(int(s["start_idx"]), int(s["end_idx"])) for s in segs] == [(s[0], s[1]) for s in ref["segments"]]
    assert np.array_equal(segs["segment_length"], np.array([s[2] for s in ref["segments"]]))
    np.testing.assert_allclose(segs["loc_error"], [s[3] for s in ref["segments"]], rtol=0, atol=1e-9)
    assert abs(r["mean_ate"] - ref["mean_ate"]) <= 1e-9 and abs(r["max_ate"] - ref["max_ate"]) <= 1e-9
    assert r["max_ate_idx"] == ref["max_ate_idx"]
    for k in ("segment_mean_ate", "segment_mean_ate_ratio"):
        assert _close(r[k], ref[k], 1e-9), (k, r[k], ref[k])


# ---- quirks ------------------------------------------------------------------------------------------------------------
def _line(n, step=1.0, axis=0):
    return [_pose((0, 0, 0, 1), [step * i if k == axis else 0.0 for k in range(3)], i, i) for i in range(n)]


def test_sequence_shorter_than_every_length_gives_nan_rpe(orc):
    gt = _line(30)
    r = orc.kitti_evaluate(gt, gt, "driving")
    assert math.isnan(r["mean_rpe"]) and len(r["tab_errors"]) == 0
    assert r["mean_ape"] == 0.0 and r["max_local_err"] == 0.0 and r["index_max_local_err"] == 0


def test_single_pose_gives_nan_local_error(orc):
    gt = _line(1)
    r = orc.kitti_evaluate(gt, gt, "indoor")
    assert math.isnan(r["mean_local_err"]) and r["index_max_local_err"] == 0 and math.isnan(r["mean_rpe"])


def test_distance_exactly_at_the_length_does_not_end_a_pair(orc):
    gt = _line(40)   # dist[i] = i exactly
    r = orc.kitti_evaluate(gt, gt, (10.0,))
    ref = np_kitti(gt, gt, (10.0,))
    # from first frame 0 the pair ends at 11 (dist 10 is not > 10), from 10 at 21, from 20 at 31; 30 has none
    assert ref["pairs"] == [(0, 11), (10, 21), (20, 31)]
    assert len(r["tab_errors"]) == 3


def test_local_error_ties_resolve_to_the_first_index(orc):
    gt = _line(8)
    # local errors 0.5 at i = 3, 4, 6 and 7: the first one is reported
    est = [_pose((0, 0, 0, 1), (x, 0, 0), i, i) for i, x in enumerate([0, 1, 2, 3.5, 4, 5, 6.5, 7])]
    r = orc.kitti_evaluate(gt, est, "indoor")
    assert r["max_local_err"] == 0.5 and r["index_max_local_err"] == 3


def test_five_pose_segment_is_skipped_but_advances_the_chain(orc):
    # steps: 4 steps of 3 m (a 5-pose segment closes at dist 12 > 10), then 1 m steps
    xs = [0, 3, 6, 9, 12] + [12 + k for k in range(1, 30)]
    gt = [_pose((0, 0, 0, 1), (x, 0, 0), i, i) for i, x in enumerate(xs)]
    rng = np.random.default_rng(5)
    est = perturbed(rng, gt, rot=0.0, tr=0.05)
    r = orc.trajectory_metrics(gt, est, 10.0)
    ref = np_metrics(gt, est, 10.0)
    starts = [(int(s["start_idx"]), int(s["end_idx"])) for s in r["segments"]]
    assert starts == [(s[0], s[1]) for s in ref["segments"]]
    assert starts[0][0] == 4   # [0, 4] (5 poses) was skipped; the next segment starts where it ended


def test_no_counted_segment_gives_nan_segment_means_and_zero_ate_gives_index_minus_one(orc):
    gt = _line(8)
    r = orc.trajectory_metrics(gt, gt, 100.0)
    assert r["num_segments"] == 0 and math.isnan(r["segment_mean_ate"]) and math.isnan(r["segment_mean_ate_ratio"])
    assert r["max_ate"] == 0.0 and r["max_ate_idx"] == -1 and r["mean_ate"] == 0.0


def test_rank_deficient_procrustes_is_finite_and_zero_gives_identity(orc):
    gt = _line(12)
    still = [_pose((0, 0, 0, 1), (5.0, -2.0, 1.0), i, i) for i in range(12)]   # stationary estimate: M = 0
    r = orc.trajectory_metrics(gt, still, 4.0)
    assert np.array_equal(r["quat"], [0, 0, 0, 1])
    ref = np_metrics(gt, still, 4.0)
    assert abs(r["mean_ate"] - ref["mean_ate"]) <= 1e-12 and abs(r["max_ate"] - ref["max_ate"]) <= 1e-12
    shifted = [_pose((0, 0, 0, 1), (0.0, 1.0 * i, 3.0), i, i) for i in range(12)]   # both straight: rank 1
    r = orc.trajectory_metrics(gt, shifted, 4.0)
    assert r["max_ate"] <= 1e-12 and all(np.isfinite(r["segments"]["loc_error"]) & (r["segments"]["loc_error"] <= 1e-12))
    u, v = np.zeros(9), np.zeros(9)
    orc.fn("svd3")(np.zeros(9).ctypes.data, u.ctypes.data, v.ctypes.data)
    assert np.array_equal(u, np.eye(3).ravel()) and np.array_equal(v, np.eye(3).ravel())


def test_svd3_against_numpy(orc):
    rng = np.random.default_rng(9)
    for k in range(200):
        A = rng.normal(size=(3, 3)) * 10.0 ** rng.uniform(-3, 3)
        if k % 4 == 1:
            A[:, 2] = 0.0
        if k % 4 == 2:
            A = np.outer(rng.normal(size=3), rng.normal(size=3))
        u, v = np.zeros(9), np.zeros(9)
        a = np.ascontiguousarray(A)
        orc.fn("svd3")(a.ctypes.data, u.ctypes.data, v.ctypes.data)
        U, V = u.reshape(3, 3), v.reshape(3, 3)
        np.testing.assert_allclose(U.T @ U, np.eye(3), atol=1e-12)
        np.testing.assert_allclose(V.T @ V, np.eye(3), atol=1e-12)
        S = U.T @ A @ V
        s = np.linalg.svd(A, compute_uv=False)
        np.testing.assert_allclose(np.diag(S), s, atol=1e-12 * s[0])
        np.testing.assert_allclose(S - np.diag(np.diag(S)), 0, atol=1e-12 * s[0])


def test_reference_unit_test_rigid_transform_scores_zero(orc):
    rng = np.random.default_rng(1234)
    gt = [_pose(_unit_quat(rng), rng.uniform(-1, 1, 3) * 100, i, i) for i in range(1000)]
    q, t = _unit_quat(rng), rng.uniform(-1, 1, 3)
    R = _R(q)
    est = [_pose(np.zeros(4), R @ np.array(p.tr[:]) + t, p.dest_timestamp, p.dest_frame_id) for p in gt]
    for e, p in zip(est, gt):   # the rotation part of rigid_transform * pose
        qa, qb = q, np.array(p.quat[:])
        w = qa[3] * qb[3] - qa[:3] @ qb[:3]
        v = qa[3] * qb[:3] + qb[3] * qa[:3] + np.cross(qa[:3], qb[:3])
        e.quat[:] = tuple(np.append(v, w) / np.linalg.norm(np.append(v, w)))
    m = orc.trajectory_metrics(gt, est, 1000.0)
    for k in ("max_ate", "mean_ate", "segment_mean_ate", "segment_mean_ate_ratio"):
        assert m[k] <= 1e-12, (k, m[k])
    k = orc.kitti_evaluate(gt, gt, "driving")
    assert k["mean_ape"] <= 1e-12 and k["max_local_err"] == 0.0


def test_ctypes_layouts_match_the_header():
    # offsets of include/cticp.h's structs as a C compiler lays them out (doubles and int64 only: no padding)
    assert C.sizeof(abi.KittiErrors) == 48
    assert C.sizeof(abi.TrajSegment) == 88 and abi.TrajSegment.quat.offset == 32 and abi.TrajSegment.tr.offset == 64
    assert C.sizeof(abi.TrajMetrics) == 112 and abi.TrajMetrics.num_segments.offset == 48
    assert abi.TrajMetrics.quat.offset == 56 and abi.TrajMetrics.tr.offset == 88
    assert abi.traj_segment_dtype().itemsize == C.sizeof(abi.TrajSegment)
    import ct_icp_b200
    eng = ct_icp_b200.engine()
    for name, cls in (("cticp_kitti_errors", abi.KittiErrors), ("cticp_traj_segment", abi.TrajSegment),
                      ("cticp_traj_metrics", abi.TrajMetrics)):
        assert eng.fn("abi_sizeof")(name.encode()) == C.sizeof(cls), name
