"""cticp_icp_register_batch_ex: B independent CERES / ROBUST registrations against one map in one persistent launch of
the Levenberg-Marquardt kernel, each problem on its own group of CTAs separated by barriers of that group alone.

Contract under test (include/cticp.h): when the problems fit the device with the CTAs a solo call would give each —
Σ (1 + ⌈(n_b + 16) / 8⌉) <= 132 co-resident CTAs on an H100 — every result is bit-identical to cticp_icp_register's;
an oversubscribed batch differs from solo by summation order only and is bit-reproducible from run to run. Problems that
stop after different numbers of ICP iterations and LM evaluations share one launch.
"""

import ctypes as C

import numpy as np
import pytest

from conftest import frame_diff, get_sequence
from ct_icp_b200 import CticpError
from ct_icp_b200 import _abi as abi

pytestmark = pytest.mark.gpu

POSE_TOL = 1e-4   # the CERES parity tests' pose tolerance against the CPU oracle (m, rad)


def _map_options(b):
    o = b.legacy_map_options(1.0, 20, 0.1)
    o.capacity_voxels = 1 << 18
    return o


def _three_level_options(b):
    """three resolutions with per-voxel normals and the sensor-side normal filter (select_valid_normals_direction)"""
    m = b.default_map_options()
    m.num_resolutions = 3
    for i, (res, md) in enumerate(((0.5, 0.05), (1.0, 0.1), (2.0, 0.2))):
        m.resolutions[i].resolution = res
        m.resolutions[i].max_num_points = 30
        m.resolutions[i].min_distance_between_points = md
    m.capacity_voxels = 1 << 18
    m.select_valid_normals_direction = 1
    return m


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
    assert len(kp) >= 2200
    return map_xyz, kp, frame, traj[-1]


@pytest.fixture(scope="module")
def emap(eng, case):
    m = eng.voxel_map(_map_options(eng))
    m.insert(case[0])
    return m


@pytest.fixture(scope="module")
def emap_normals(eng, case):
    """the same points inserted from a sensor origin into a map that keeps oriented per-voxel normals"""
    m = eng.voxel_map(_three_level_options(eng))
    m.insert(case[0], np.array(case[3].end_pose.tr))
    return m


def _ceres_options(b, loss="CAUCHY", iters=4):
    io = b.default_icp_options()
    io.solver = abi.SOLVER["CERES"]
    io.loss_function = abi.LOSS[loss]
    io.min_number_neighbors = 10
    io.num_iters_icp = iters
    io.ls_max_num_iters = 5
    io.threshold_orientation_norm = 1e-9     # run every ICP iteration
    io.threshold_translation_norm = 1e-9
    return io


def _robust_options(b):
    io = b.default_icp_options()
    io.solver = abi.SOLVER["ROBUST"]
    io.num_iters_icp = 4
    io.max_num_residuals = -1
    io.weight_alpha = 0.9
    io.weight_neighborhood = 0.1
    io.min_number_neighbors = 8
    io.max_number_neighbors = 20
    io.loss_function = abi.LOSS["CAUCHY"]
    io.ls_max_num_iters = 8
    io.ls_sigma = 0.1
    io.max_dist_to_plane_ct_icp = 0.5
    io.threshold_linearity = 0.6
    io.threshold_planarity = 0.8
    io.outlier_distance = 0.8
    io.use_barycenter = 1
    io.use_lines = 1
    return io


def _distance_based():
    st = abi.StrategyOptions(abi.STRATEGY["DISTANCE_BASED_STRATEGY"], 20, 8)
    st.radius_min, st.radius_max, st.exponent, st.distance_max = 0.1, 1.2, 1.0, 60.0
    return st


def _motion_model(b):
    mm = b.default_odometry_options().default_motion_model
    mm.beta_small_velocity = 0.0005         # exercise every regulariser
    mm.beta_orientation_consistency = 0.0005
    return mm


def _perturbed(frame, k):
    """frame moved by a few centimetres (problem k's initial guess)"""
    f = frame.copy()
    d = 0.03 * np.array([np.cos(1.3 * k), np.sin(0.7 * k), 0.3 * np.cos(2.1 * k)])
    f.begin_pose.tr = tuple(np.array(f.begin_pose.tr) + d)
    f.end_pose.tr = tuple(np.array(f.end_pose.tr) + d)
    return f


def _with_world(orc, kp, frame):
    """kp with `world` at `frame`"""
    kp = kp.copy()
    out = (C.c_double * 3)()
    for i in range(len(kp)):
        raw = (C.c_double * 3)(*kp["raw"][i])
        orc.check(orc.fn("pose_transform")(C.byref(frame), raw, float(kp["timestamp"][i]), out))
        kp["world"][i] = out[:]
    return kp


def _sub(kp, j, n):
    """n keypoints spread over the whole scan (every 9th from j)"""
    return kp[j::9][:n].copy()


def _solo(m, io, kp, frame, prev, mm, st=None):
    k, f = kp.copy(), frame.copy()
    s = m.icp_register(io, k, f, prev, mm if prev is not None else None, st)
    return k, f, s


def _batch(m, io, kps, frames, prevs, mm, st=None):
    ks, fs = [k.copy() for k in kps], [f.copy() for f in frames]
    ss = m.icp_register_batch_ex(io, ks, fs, prevs, mm, st)
    return list(zip(ks, fs, ss))


def _assert_same(a, b):
    """(keypoints, frame, summary) of two runs: bit-identical"""
    ka, fa, sa = a
    kb, fb, sb = b
    assert bytes(fa) == bytes(fb)
    assert (sa.success, sa.num_residuals_used, sa.num_iters) == (sb.success, sb.num_residuals_used, sb.num_iters)
    assert ka["world"].tobytes() == kb["world"].tobytes()


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["ceres_cauchy", "ceres_distance_based", "ceres_ncn2", "robust"])
def test_batch_that_fits_is_bit_identical_to_solo(eng, case, emap, emap_normals, variant):
    _, kp, frame, prev = case
    m, st = emap, None
    if variant == "robust":
        io = _robust_options(eng)
    else:
        io = _ceres_options(eng)
        io.max_num_residuals = 150
        if variant == "ceres_distance_based":
            m, st = emap_normals, _distance_based()
        elif variant == "ceres_ncn2":
            io.num_closest_neighbors = 2
            io.max_num_residuals = 300
    mm = _motion_model(eng)
    # 4 problems of 200..240 keypoints: Σ (1 + ⌈(n + 16) / 8⌉) = 124 CTAs, every problem gets its solo grid
    sizes = (240, 200, 230, 220)
    kps = [_sub(kp, i, n) for i, n in enumerate(sizes)]
    frames = [_perturbed(frame, k) for k in range(4)]
    prev2 = prev.copy()
    prev2.end_pose.tr = tuple(np.array(prev2.end_pose.tr) + [0.05, -0.02, 0.0])
    prevs = [prev, None, prev2, prev]
    got = _batch(m, io, kps, frames, prevs, mm, st)
    for b in range(4):
        ref = _solo(m, io, kps[b], frames[b], prevs[b], mm, st)
        assert ref[2].success
        _assert_same(got[b], ref)
        assert frame_diff(got[b][1], frames[b], log=False)[0] > 1e-4   # the registration moved the pose
    # B = 1 (the full keypoint set): the solo call's grid, its result
    got1 = _batch(m, io, [kp], [frame], [prev], mm, st)
    _assert_same(got1[0], _solo(m, io, kp, frame, prev, mm, st))


def test_groups_that_stop_at_different_times(eng, case, emap):
    """One launch hosts problems that leave the loop after different numbers of ICP iterations and LM evaluations:
    a barrier count that differed between the CTAs of a group would hang or corrupt that group."""
    _, kp, frame, prev = case
    io = _ceres_options(eng, iters=6)
    io.threshold_orientation_norm = 0.05    # the converged problem stops after its first ICP iteration
    io.threshold_translation_norm = 0.05
    mm = _motion_model(eng)
    # a problem that starts at its converged pose: map points seen from the identity pose
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
    far = _perturbed(frame, 2)
    far.end_pose.tr = tuple(np.array(far.end_pose.tr) + [0.25, -0.15, 0.0])   # far from its optimum: more iterations
    # 4 + 3 + 33 + 28 + 33 + 22 = 123 CTAs: every problem gets its solo grid
    kps = [_sub(kp, 5, 6), np.zeros(0, dtype=abi.wpoint_dtype()), conv, lo, _sub(kp, 3, 240), _sub(kp, 4, 150)]
    frames = [frame, frame, f_conv, _perturbed(frame, 1), far, _perturbed(frame, 3)]
    prevs = [prev, None, None, prev, None, None]
    got = _batch(emap, io, kps, frames, prevs, mm)
    assert not got[0][2].success and not got[1][2].success      # too few keypoints; no keypoints
    for b in range(len(kps)):
        _assert_same(got[b], _solo(emap, io, kps[b], frames[b], prevs[b], mm))
    iters = [got[b][2].num_iters for b in (2, 3, 4, 5)]
    assert all(got[b][2].success for b in (2, 3, 4, 5))
    assert got[2][2].num_iters <= 1 and got[4][2].num_iters > got[2][2].num_iters, iters
    assert frame_diff(got[4][1], frames[4], log=False)[0] > 1e-2


def test_oversubscribed_batch_matches_oracle_and_repeats(orc, eng, case, emap):
    map_xyz, kp, frame, prev = case
    mo = orc.voxel_map(_map_options(orc))
    mo.insert(map_xyz)
    io = _ceres_options(eng)
    io.max_num_residuals = 700
    mm = _motion_model(eng)
    B = 8
    frames = [_perturbed(frame, k) for k in range(B)]
    kps = [_with_world(orc, kp, f) for f in frames]
    prevs = [prev] * B
    st = abi.StrategyOptions(0, 20, 8, 0)
    got = _batch(emap, io, kps, frames, prevs, mm, st)
    again = _batch(emap, io, kps, frames, prevs, mm, st)
    for b in range(B):
        _assert_same(got[b], again[b])
        io_o = _ceres_options(orc)
        io_o.max_num_residuals = 700
        ko, fo, so = _solo(mo, io_o, kps[b], frames[b], prev, _motion_model(orc), st)
        ke, fe, se = got[b]
        assert so.success and se.success
        assert so.num_residuals_used == se.num_residuals_used == 700
        dt, dr = frame_diff(fo, fe)
        assert dt < POSE_TOL and dr < POSE_TOL, (b, dt, dr)
        assert frame_diff(fe, frames[b], log=False)[0] > 1e-3    # the registration moved the pose


def test_batch_errors_leave_the_map_usable(eng, case, emap):
    _, kp, frame, prev = case
    io = _ceres_options(eng)
    io.max_num_residuals = 150
    mm = _motion_model(eng)
    kps = [_sub(kp, b, 200) for b in range(3)]
    frames = [_perturbed(frame, k) for k in range(3)]
    ref = [_solo(emap, io, kps[b], frames[b], prev, mm) for b in range(3)]

    def check_usable():
        got = _batch(emap, io, kps, frames, [prev] * 3, mm)
        for b in range(3):
            _assert_same(got[b], ref[b])

    def expect(code, options, kps_, frames_, st=None):
        with pytest.raises(CticpError) as e:
            emap.icp_register_batch_ex(options, kps_, frames_, None, None, st)
        assert e.value.code == code
        check_usable()

    # null arguments, batch outside [1, 64]
    fn = emap.b.fn("icp_register_batch_ex")
    assert fn(emap.h, None, None, 1, None, None, None, None, None, None) == abi.ERR_INVALID_ARGUMENT
    check_usable()
    expect(abi.ERR_INVALID_ARGUMENT, io, [], [])
    expect(abi.ERR_INVALID_ARGUMENT, io, [kp[:10].copy() for _ in range(65)], [frame.copy() for _ in range(65)])

    # options a solo CERES call rejects
    p2p = _ceres_options(eng)
    p2p.distance = abi.DISTANCE["POINT_TO_POINT"]
    expect(abi.ERR_UNSUPPORTED, p2p, [k.copy() for k in kps], [f.copy() for f in frames])
    ncn5 = _ceres_options(eng)
    ncn5.num_closest_neighbors = 5
    expect(abi.ERR_UNSUPPORTED, ncn5, [k.copy() for k in kps], [f.copy() for f in frames])
    st = _distance_based()
    st.radius_max = 0.0
    expect(abi.ERR_INVALID_ARGUMENT, io, [k.copy() for k in kps], [f.copy() for f in frames], st)

    # a keypoint of problem 2 outside its frame: nothing runs, no frame changes
    bad = [k.copy() for k in kps]
    bad[1]["timestamp"][17] = frame.end_pose.dest_timestamp + 1.0
    fs = [f.copy() for f in frames]
    with pytest.raises(CticpError) as e:
        emap.icp_register_batch_ex(io, bad, fs, [prev] * 3, mm)
    assert e.value.code == abi.ERR_TIMESTAMP
    assert all(bytes(a) == bytes(b) for a, b in zip(fs, frames))
    check_usable()

    # solver GN through the _ex entry: the GN batch
    gn = eng.default_icp_options()
    gn.solver = abi.SOLVER["GN"]
    gn.min_number_neighbors = 10
    gn.num_iters_icp = 8
    ks1, fs1 = [k.copy() for k in kps], [f.copy() for f in frames]
    ks2, fs2 = [k.copy() for k in kps], [f.copy() for f in frames]
    s1 = emap.icp_register_batch(gn, ks1, fs1, [prev] * 3, mm)
    s2 = emap.icp_register_batch_ex(gn, ks2, fs2, [prev] * 3, mm, _distance_based())
    for b in range(3):
        _assert_same((ks1[b], fs1[b], s1[b]), (ks2[b], fs2[b], s2[b]))
