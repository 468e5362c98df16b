"""cticp_icp_register_batch: B independent Gauss-Newton registrations against one map in one persistent launch.

Contract under test (include/cticp.h): when the problems fit the device together with the CTAs a solo call would give
each — Σ (1 + ⌈(n_b + 16) / 8⌉) <= 132 co-resident CTAs on an H100 — every result is bit-identical to cticp_icp_register's;
an oversubscribed batch differs from solo by summation order only and is bit-reproducible from run to run.
"""

import ctypes as C

import numpy as np
import pytest

from conftest import frame_diff, get_sequence
from ct_icp_b200 import CticpError
from ct_icp_b200 import _abi as abi

pytestmark = pytest.mark.gpu


def _map_options(b):
    o = b.legacy_map_options(1.0, 20, 0.1)
    o.capacity_voxels = 1 << 18
    return o


@pytest.fixture(scope="module")
def case(orc):
    """Map from HDL-64 frames 0..2 at the oracle's poses; frame 3's keypoints (1.0 m grid), its initial frame, the
    previous frame."""
    seq = get_sequence("hdl64", 4)
    o = orc.default_odometry_options()
    o.ct_icp_options.solver = abi.SOLVER["GN"]
    o.ct_icp_options.min_number_neighbors = 10
    o.map_options = orc.legacy_map_options(1.0, 20, 0.1)
    o.debug_print = 0
    od = orc.odometry(o)
    for s in seq[:3]:
        assert od.RegisterFrame(s["xyz"], s["t"], s["frame_idx"]).success
    map_xyz, _ = od.GetMapPointer().export(0)
    s = seq[3]
    idx = orc.grid_sample_indices(s["xyz"], 1.0)
    kp = np.zeros(len(idx), dtype=abi.wpoint_dtype())
    kp["raw"] = s["xyz"][idx]
    kp["timestamp"] = s["t"][idx]
    traj = od.Trajectory()
    frame = traj[-1].copy()
    frame.begin_pose = traj[-1].end_pose.copy()
    frame.begin_pose.dest_timestamp = float(s["t"].min())
    frame.end_pose.dest_timestamp = float(s["t"].max())
    assert len(kp) >= 2000
    return map_xyz, kp, frame, traj[-1]


@pytest.fixture(scope="module")
def emap(eng, case):
    m = eng.voxel_map(_map_options(eng))
    m.insert(case[0])
    return m


def _gn_options(b, iters=8):
    io = b.default_icp_options()
    io.solver = abi.SOLVER["GN"]
    io.min_number_neighbors = 10
    io.num_iters_icp = iters
    return io


def _perturbed(frame, k):
    """frame moved by a few centimetres (problem k's initial guess)"""
    f = frame.copy()
    d = 0.03 * np.array([np.cos(1.3 * k), np.sin(0.7 * k), 0.3 * np.cos(2.1 * k)])
    f.begin_pose.tr = tuple(np.array(f.begin_pose.tr) + d)
    f.end_pose.tr = tuple(np.array(f.end_pose.tr) + d)
    return f


def _with_world(orc, kp, frame):
    """kp with `world` at `frame` (the input world points the reference's first neighborhood search starts from)"""
    kp = kp.copy()
    out = (C.c_double * 3)()
    for i in range(len(kp)):
        raw = (C.c_double * 3)(*kp["raw"][i])
        orc.check(orc.fn("pose_transform")(C.byref(frame), raw, float(kp["timestamp"][i]), out))
        kp["world"][i] = out[:]
    return kp


def _sub(kp, j, n):
    """n keypoints spread over the whole scan (every 9th from j): a consecutive run would sit in a few rings"""
    return kp[j::9][:n].copy()


def _solo(m, io, kp, frame, prev, mm):
    k, f = kp.copy(), frame.copy()
    s = m.icp_register(io, k, f, prev, mm if prev is not None else None)
    return k, f, s


def _assert_same(a, b):
    """(keypoints, frame, summary) of two runs: bit-identical"""
    ka, fa, sa = a
    kb, fb, sb = b
    assert bytes(fa) == bytes(fb)
    assert (sa.success, sa.num_residuals_used, sa.num_iters) == (sb.success, sb.num_residuals_used, sb.num_iters)
    assert ka["world"].tobytes() == kb["world"].tobytes()


def _batch(m, io, kps, frames, prevs, mm):
    ks, fs = [k.copy() for k in kps], [f.copy() for f in frames]
    ss = m.icp_register_batch(io, ks, fs, prevs, mm)
    return list(zip(ks, fs, ss))


# ---------------------------------------------------------------------------------------------------------------
def test_batch_that_fits_is_bit_identical_to_solo(eng, case, emap):
    _, kp, frame, prev = case
    io = _gn_options(eng)
    mm = eng.default_odometry_options().default_motion_model
    # 4 problems of 200..240 keypoints: Σ (1 + ⌈(n + 16) / 8⌉) = 124 CTAs, every problem gets its solo grid
    sizes = (240, 200, 230, 220)
    kps = [_sub(kp, i, n) for i, n in enumerate(sizes)]
    frames = [_perturbed(frame, k) for k in range(4)]
    prev2 = prev.copy()
    prev2.end_pose.tr = tuple(np.array(prev2.end_pose.tr) + [0.05, -0.02, 0.0])
    prevs = [prev, None, prev2, prev]
    got = _batch(emap, io, kps, frames, prevs, mm)
    for b in range(4):
        ref = _solo(emap, io, kps[b], frames[b], prevs[b], mm)
        assert ref[2].success
        _assert_same(got[b], ref)
    # B = 1 (the full keypoint set): the solo call's grid, its result
    got1 = _batch(emap, io, [kp], [frame], [prev], mm)
    _assert_same(got1[0], _solo(emap, io, kp, frame, prev, mm))


def test_oversubscribed_batch_matches_oracle_and_repeats(orc, eng, case, emap):
    map_xyz, kp, frame, prev = case
    mo = orc.voxel_map(_map_options(orc))
    mo.insert(map_xyz)
    io = _gn_options(eng)
    mm = eng.default_odometry_options().default_motion_model
    B = 8
    frames = [_perturbed(frame, k) for k in range(B)]
    kps = [_with_world(orc, kp, f) for f in frames]
    prevs = [prev] * B
    got = _batch(emap, io, kps, frames, prevs, mm)
    again = _batch(emap, io, kps, frames, prevs, mm)
    for b in range(B):
        _assert_same(got[b], again[b])
        ko, fo, so = _solo(mo, _gn_options(orc), kps[b], frames[b], prev, orc.default_odometry_options().default_motion_model)
        ke, fe, se = got[b]
        assert so.success and se.success
        assert so.num_residuals_used == se.num_residuals_used
        dt, dr = frame_diff(fo, fe)
        assert dt < 1e-6 and dr < 1e-6, (b, dt, dr)
        assert frame_diff(fe, frames[b], log=False)[0] > 1e-3    # the registration moved the pose
        assert np.abs(ko["world"] - ke["world"]).max() < 1e-5


def test_mixed_outcomes_in_one_batch(eng, case, emap):
    _, kp, frame, prev = case
    io = _gn_options(eng, iters=20)
    io.threshold_orientation_norm = 1e-2   # the converged problem must stop after its first step
    mm = eng.default_odometry_options().default_motion_model
    ordinary = _sub(kp, 3, 240)
    # a problem that starts at its converged pose: map points seen from the identity pose (first step ~0)
    map_xyz = case[0]
    conv = np.zeros(240, dtype=abi.wpoint_dtype())
    conv["raw"] = map_xyz[:: max(1, len(map_xyz) // 240)][:240]
    conv["timestamp"] = 0.05
    f_conv = abi.Frame()
    f_conv.begin_pose = abi.Pose.make(dest_timestamp=0.0)
    f_conv.end_pose = abi.Pose.make(dest_timestamp=0.1)
    # float64 coordinates that float32 does not represent: the problem needs the residual plane
    lo = _sub(kp, 2, 200)
    lo["raw"] += 1e-7 * np.random.default_rng(3).uniform(-1.0, 1.0, size=(len(lo), 3))
    assert np.any(lo["raw"].astype(np.float32).astype(np.float64) != lo["raw"])
    # 10 + 3 + 33 + 28 + 33 + 22 = 129 CTAs: every problem gets its solo grid
    kps = [_sub(kp, 5, 50), np.zeros(0, dtype=abi.wpoint_dtype()), conv, lo, ordinary, _sub(kp, 4, 150)]
    frames = [frame, frame, f_conv, _perturbed(frame, 1), _perturbed(frame, 2), _perturbed(frame, 3)]
    prevs = [prev, None, None, prev, prev, None]
    got = _batch(emap, io, kps, frames, prevs, mm)
    assert not got[0][2].success and not got[1][2].success
    assert got[2][2].success and got[2][2].num_iters == 1
    for b in range(len(kps)):
        _assert_same(got[b], _solo(emap, io, kps[b], frames[b], prevs[b], mm))
    for b in (3, 4):
        assert got[b][2].success and frame_diff(got[b][1], frames[b], log=False)[0] > 1e-3


def test_batch_errors_leave_the_map_usable(eng, case, emap):
    _, kp, frame, prev = case
    io = _gn_options(eng)
    mm = eng.default_odometry_options().default_motion_model
    kps = [_sub(kp, b, 200) for b in range(3)]
    frames = [_perturbed(frame, k) for k in range(3)]
    ref = [_solo(emap, io, kps[b], frames[b], prev, mm) for b in range(3)]

    def check_usable():
        got = _batch(emap, io, kps, frames, [prev] * 3, mm)
        for b in range(3):
            _assert_same(got[b], ref[b])

    # a keypoint of problem 2 outside its frame: nothing runs, no frame changes
    bad = [k.copy() for k in kps]
    bad[1]["timestamp"][17] = frame.end_pose.dest_timestamp + 1.0
    fs = [f.copy() for f in frames]
    with pytest.raises(CticpError) as e:
        emap.icp_register_batch(io, bad, fs, [prev] * 3, mm)
    assert e.value.code == abi.ERR_TIMESTAMP
    assert all(bytes(a) == bytes(b) for a, b in zip(fs, frames))
    check_usable()

    ceres = _gn_options(eng)
    ceres.solver = abi.SOLVER["CERES"]
    with pytest.raises(CticpError) as e:
        emap.icp_register_batch(ceres, [k.copy() for k in kps], [f.copy() for f in frames], None, None)
    assert e.value.code == abi.ERR_UNSUPPORTED
    check_usable()

    with pytest.raises(CticpError) as e:
        emap.icp_register_batch(io, [], [], None, None)
    assert e.value.code == abi.ERR_INVALID_ARGUMENT
    check_usable()

    many = [kp[:10].copy() for _ in range(65)]
    with pytest.raises(CticpError) as e:
        emap.icp_register_batch(io, many, [frame.copy() for _ in range(65)], None, None)
    assert e.value.code == abi.ERR_INVALID_ARGUMENT
    check_usable()
