"""World clouds and slam::SamplePointsInGrid on the device (cticp_sample_points_in_grid, cticp_world_cloud_*): the
one-shot function against the CPU restatement (tests/oracle_grid), the incremental cloud against the one-shot function
over the concatenation of its inputs, world points along a trajectory and from an odometry, rejections, capacity,
refusals and repeatability."""
import ctypes as C

import numpy as np
import pytest

from ct_icp_b200 import _abi as abi
from ct_icp_b200._binding import CticpError
from conftest import get_sequence
from grid_numpy import sample_points_in_grid as np_sample
from oracle_grid_lib import grid_oracle

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def _cloud(n, seed, scale=3.0):
    return np.random.default_rng(seed).uniform(-scale, scale, (n, 3))


def _export_all(wc):
    pts, src = wc.export(np.float64, with_timestamps=True, with_source_index=True)
    return pts, src


@pytest.mark.parametrize("n", [0, 1, 2, 1000, 100_000])
@pytest.mark.parametrize("npv", [0, 1, 2, 5])
def test_one_shot_against_the_restatement(eng, n, npv):
    xyz = _cloud(n, 7 + n)
    for mx in (-7, -1, 0, 1, 37, 10 ** 9):
        got = eng.sample_points_in_grid(xyz, 0.5, npv, mx)
        np.testing.assert_array_equal(got, grid_oracle().sample_points_in_grid(xyz, 0.5, npv, mx))


def test_one_shot_faces_and_truncated_voxel_zero(eng):
    rng = np.random.default_rng(11)
    faces = np.concatenate([rng.integers(-50, 50, (20000, 3)) * 0.1, rng.uniform(-0.25, 0.25, (5000, 3))])
    for npv in (0, 1, 3):
        np.testing.assert_array_equal(eng.sample_points_in_grid(faces, 0.1, npv), np_sample(faces, 0.1, npv))
        np.testing.assert_array_equal(eng.sample_points_in_grid(faces, 0.1, npv),
                                      grid_oracle().sample_points_in_grid(faces, 0.1, npv))


def test_one_shot_8m_points(eng):
    xyz = _cloud(8_000_000, 8, scale=40.0)
    for npv in (1, 4):
        got = eng.sample_points_in_grid(xyz, 0.2, npv)
        np.testing.assert_array_equal(got, grid_oracle().sample_points_in_grid(xyz, 0.2, npv))


@pytest.mark.parametrize("npv", [1, 3])
@pytest.mark.parametrize("calls", [1, 2, 7, 64])
def test_incremental_equals_one_shot(eng, npv, calls):
    rng = np.random.default_rng(calls * 10 + npv)
    n = 60_000
    xyz = rng.uniform(-8, 8, (n, 3))
    t = rng.uniform(0, 10, n)
    cuts = np.sort(rng.integers(0, n + 1, calls - 1))
    cuts[: min(2, len(cuts))] = cuts[0] if len(cuts) else 0      # empty calls
    parts = np.split(np.arange(n), cuts)
    for mx in (-1, 5000):
        wc = eng.world_cloud(0.25, npv, mx)
        submitted = kept = 0
        for p in parts:
            st = wc.add(xyz[p], t[p])
            assert st.submitted == len(p) and st.rejected == 0
            submitted += st.submitted
            kept += st.kept
        ref = np_sample(xyz, 0.25, npv, mx)
        pts, src = _export_all(wc)
        np.testing.assert_array_equal(src, ref)
        assert pts[:, :3].tobytes() == xyz[ref.astype(np.int64)].tobytes()
        assert pts[:, 3].tobytes() == t[ref.astype(np.int64)].tobytes()
        assert wc.num_points() == len(ref) and kept == len(np_sample(xyz, 0.25, npv))
        assert wc.num_voxels() == len(np_sample(xyz, 0.25, 1))
        wc.close()


def test_without_timestamps_and_float32(eng):
    xyz = _cloud(20000, 4).astype(np.float32)
    wc = eng.world_cloud(0.3, 2)
    wc.add(xyz[:7000])
    wc.add(torch.from_numpy(xyz[7000:]).cuda())
    torch.cuda.synchronize()
    pts, src = _export_all(wc)
    ref = np_sample(xyz.astype(np.float64), 0.3, 2)
    np.testing.assert_array_equal(src, ref)
    assert (pts[:, 3] == 0.0).all()
    assert pts[:, :3].tobytes() == xyz.astype(np.float64)[ref.astype(np.int64)].tobytes()
    f32 = wc.export(np.float32)
    np.testing.assert_array_equal(f32, xyz[ref.astype(np.int64)])


def _trajectory(eng, nframes=8):
    frames = []
    for k in range(nframes):
        f = abi.Frame()
        f.begin_pose = abi.Pose.make(quat=[0, 0, np.sin(0.05 * k), np.cos(0.05 * k)], tr=[2.0 * k, 0.3 * k, 0],
                                     dest_timestamp=k * 0.1, dest_frame_id=k)
        f.end_pose = abi.Pose.make(quat=[0, 0, np.sin(0.05 * k + 0.04), np.cos(0.05 * k + 0.04)],
                                   tr=[2.0 * k + 1.9, 0.3 * k + 0.25, 0.01], dest_timestamp=k * 0.1 + 0.1, dest_frame_id=k)
        frames.append(f)
    return eng.continuous_trajectory(frames)


@pytest.mark.parametrize("mode", ["timestamp", "segments"])
def test_along_a_trajectory(eng, mode):
    rng = np.random.default_rng(5)
    traj = _trajectory(eng)
    per = 20000
    scans = []
    for k in range(8):
        xyz = rng.uniform(-20, 20, (per, 3))
        t = k * 0.1 + rng.uniform(0, 0.1, per)
        scans.append((xyz, t))
    xyz_all = np.concatenate([s[0] for s in scans])
    t_all = np.concatenate([s[1] for s in scans])
    ends = np.cumsum([per] * 8)
    segs_all = (ends, np.arange(8)) if mode == "segments" else None
    w = traj.transform(xyz_all, t_all, segments=segs_all, dtype=np.float64)
    ref = np_sample(w, 0.2, 2)
    exports = []
    for path in ("host64", "host32", "device64", "unaligned"):
        wc = eng.world_cloud(0.2, 2)
        for k, (xyz, t) in enumerate(scans):
            seg = (np.array([per]), np.array([k])) if mode == "segments" else None
            if path == "host64":
                wc.add(xyz, t, trajectory=traj, segments=seg)
            elif path == "host32":   # float32 records: the trajectory reads them in fp64 as it would
                x32 = xyz.astype(np.float32)
                wc.add(x32, t, trajectory=traj, segments=seg)
            elif path == "device64":
                wc.add(torch.from_numpy(xyz).cuda(), torch.from_numpy(t).cuda(), trajectory=traj, segments=seg)
            else:   # packed records, x at offset 1, t at offset 25
                rec = np.zeros(per, dtype=np.dtype({"names": ["x", "y", "z", "t"], "formats": ["<f8"] * 4,
                                                    "offsets": [1, 9, 17, 25], "itemsize": 33}))
                rec["x"], rec["y"], rec["z"], rec["t"] = xyz[:, 0], xyz[:, 1], xyz[:, 2], t
                wc.add_records(rec, trajectory=traj, segments=seg)
        torch.cuda.synchronize()
        pts, src = _export_all(wc)
        if path == "host32":
            x32 = np.concatenate([s[0].astype(np.float32) for s in scans])
            w32 = traj.transform(x32, t_all, segments=segs_all, dtype=np.float64)
            ref32 = np_sample(w32, 0.2, 2)
            np.testing.assert_array_equal(src, ref32)
            assert pts[:, :3].tobytes() == w32[ref32.astype(np.int64)].tobytes()
        else:
            np.testing.assert_array_equal(src, ref)
            assert pts[:, :3].tobytes() == w[ref.astype(np.int64)].tobytes()
            assert pts[:, 3].tobytes() == t_all[ref.astype(np.int64)].tobytes()
            exports.append(pts.tobytes() + src.tobytes())
        wc.close()
    assert len(set(exports)) == 1


def test_from_odometry(eng):
    o = eng.default_odometry_options()
    o.ct_icp_options.solver = abi.SOLVER["GN"]
    o.ct_icp_options.min_number_neighbors = 10
    o.map_options = eng.legacy_map_options(1.0, 20, 0.1)
    o.init_num_frames = 3
    o.debug_print = 0
    o.ct_icp_options.debug_print = 0
    od = eng.odometry(o)
    a, b = eng.world_cloud(0.3, 2), eng.world_cloud(0.3, 2)
    for s in get_sequence("small16", 6):
        sm = od.RegisterFrame(s["xyz"], s["t"], s["frame_idx"])
        assert sm.success, sm.error_message
        st = a.add_odometry(od)
        w = od.points_device(abi.POINTS_ALL_CORRECTED, world=True, dtype=torch.float64, with_timestamps=True)
        b.add(w[:, :3], w[:, 3])
        assert st.submitted == w.shape[0]
    torch.cuda.synchronize()
    pa, sa = _export_all(a)
    pb, sb = _export_all(b)
    assert pa.tobytes() == pb.tobytes() and sa.tobytes() == sb.tobytes() and len(pa) > 0
    od.close()


def test_rejections(eng):
    xyz = _cloud(30000, 9)
    bad = np.random.default_rng(1).choice(30000, 300, replace=False)
    xyz[bad[:100], 0] = np.nan
    xyz[bad[100:200], 1] = -np.inf
    xyz[bad[200:], 2] = 0.5 * 2.0 ** 20 * (1 + np.random.default_rng(2).random(100))   # voxel coordinate >= 2^20 at 0.5
    wc = eng.world_cloud(0.5, 3)
    st1 = wc.add(xyz[:12345])
    st2 = wc.add(xyz[12345:])
    assert st1.rejected + st2.rejected == 300
    _, src = _export_all(wc)
    ref = np_sample(xyz, 0.5, 3)
    np.testing.assert_array_equal(src, ref)
    keep = np.setdiff1d(np.arange(30000), bad)
    np.testing.assert_array_equal(src, keep[np_sample(xyz[keep], 0.5, 3).astype(np.int64)])


def test_capacity_leaves_the_cloud_unchanged(eng):
    xyz = _cloud(50000, 12, scale=10.0)
    wc = eng.world_cloud(0.5, 2, capacity_voxels=5000, capacity_points=8000)
    wc.add(xyz[:1000])
    before = _export_all(wc)
    nv, npts = wc.num_voxels(), wc.num_points()
    with pytest.raises(CticpError) as e:
        wc.add(xyz[1000:])
    assert e.value.code == abi.ERR_CAPACITY
    after = _export_all(wc)
    assert before[0].tobytes() == after[0].tobytes() and before[1].tobytes() == after[1].tobytes()
    assert (wc.num_voxels(), wc.num_points()) == (nv, npts)
    wc.add(xyz[1000:1500])   # still consistent: as if the refused call never happened (source indices continue)
    _, src = _export_all(wc)
    np.testing.assert_array_equal(src, np_sample(xyz[:1500], 0.5, 2))
    wc.clear()
    assert wc.num_points() == 0 and wc.num_voxels() == 0
    wc.add(xyz[:3000])
    _, src = _export_all(wc)
    np.testing.assert_array_equal(src, np_sample(xyz[:3000], 0.5, 2))


def test_refusals_change_nothing(eng):
    xyz = _cloud(5000, 13)
    for g in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(CticpError) as e:
            eng.world_cloud(g)
        assert e.value.code == abi.ERR_INVALID_ARGUMENT
        with pytest.raises(CticpError) as e:
            eng.sample_points_in_grid(xyz, g)
        assert e.value.code == abi.ERR_INVALID_ARGUMENT
    for npv in (65, -1):
        with pytest.raises(CticpError) as e:
            eng.world_cloud(0.5, npv)
        assert e.value.code == abi.ERR_UNSUPPORTED
    traj = _trajectory(eng)
    wc = eng.world_cloud(0.5, 2)
    wc.add(xyz[:2000], np.zeros(2000))
    before = _export_all(wc)
    f = eng.fn("world_cloud_add")
    view = abi.CloudView(None, 10, 32, 0, abi.DTYPE["float64"], 24, abi.DTYPE["float64"], 0)
    assert f(wc.h, None, C.byref(view), None, None, 0, None) == abi.ERR_INVALID_ARGUMENT    # null data
    assert f(None, None, C.byref(view), None, None, 0, None) == abi.ERR_INVALID_ARGUMENT
    assert f(wc.h, None, None, None, None, 0, None) == abi.ERR_INVALID_ARGUMENT
    rec = np.zeros(10, dtype=[("x", "<f8"), ("y", "<f8"), ("z", "<f8"), ("t", "<f8")])
    for xdt, tdt, step in ((abi.DTYPE["int32"], 8, 32), (8, 9, 32), (8, 8, 16)):
        view = abi.CloudView(rec.ctypes.data, 10, step, 0, xdt, 24, tdt, 0)
        assert f(wc.h, None, C.byref(view), None, None, 0, None) == abi.ERR_INVALID_ARGUMENT
    norec = np.zeros(10, dtype=[("x", "<f8"), ("y", "<f8"), ("z", "<f8")])
    with pytest.raises(CticpError):   # a trajectory needs timestamps
        wc.add_records(norec, trajectory=traj)
    with pytest.raises(CticpError):   # a frame above every pose's
        wc.add(xyz[:10], np.zeros(10), trajectory=traj, segments=(np.array([10]), np.array([99])))
    with pytest.raises(CticpError):   # segment ends that do not end at the point count
        wc.add(xyz[:10], np.zeros(10), trajectory=traj, segments=(np.array([9]), np.array([0])))
    with pytest.raises(CticpError):   # segments without a trajectory
        wc.add(xyz[:10], np.zeros(10), segments=(np.array([10]), np.array([0])))
    # device pointers: host memory, and a buffer shorter than described
    host = np.zeros((10, 3))
    scan = abi.DeviceScan(host.ctypes.data, 24, None, 0, 10, abi.DTYPE["float64"], 0)
    with pytest.raises(CticpError) as e:
        wc.add_device(scan)
    assert e.value.code == abi.ERR_INVALID_ARGUMENT
    d = torch.zeros((10, 3), dtype=torch.float64, device="cuda")
    scan = abi.DeviceScan(d.data_ptr(), 24, None, 0, 1 << 20, abi.DTYPE["float64"], 0)
    with pytest.raises(CticpError) as e:
        wc.add_device(scan)
    assert e.value.code == abi.ERR_INVALID_ARGUMENT
    after = _export_all(wc)
    assert before[0].tobytes() == after[0].tobytes() and before[1].tobytes() == after[1].tobytes()
    # export refusals leave the sink untouched
    sink_buf = np.full((wc.num_points(), 4), 7.0)
    bad = abi.CloudSink(sink_buf.ctypes.data, len(sink_buf), 32, 0, abi.DTYPE["int32"], 24, 8, 1)
    assert eng.fn("world_cloud_export")(wc.h, C.byref(bad), None) == abi.ERR_INVALID_ARGUMENT
    bad = abi.CloudSink(sink_buf.ctypes.data, len(sink_buf), 32, 0, 8, 24, 8, 0)   # world = 0
    assert eng.fn("world_cloud_export")(wc.h, C.byref(bad), None) == abi.ERR_INVALID_ARGUMENT
    assert (sink_buf == 7.0).all()
    dsink = abi.CloudSink(sink_buf.ctypes.data, len(sink_buf), 32, 0, 8, 24, 8, 1)   # host memory as a device sink
    assert eng.fn("world_cloud_export_device")(wc.h, C.byref(dsink), None, None) == abi.ERR_INVALID_ARGUMENT
    assert (sink_buf == 7.0).all()


def test_repeatable_and_device_export(eng):
    rng = np.random.default_rng(21)
    xyz = torch.from_numpy(rng.uniform(-30, 30, (400_000, 3))).cuda()
    t = torch.from_numpy(rng.uniform(0, 1, 400_000)).cuda()
    outs = []
    for _ in range(2):
        wc = eng.world_cloud(0.2, 4)
        for k in range(0, 400_000, 50_000):
            wc.add(xyz[k:k + 50_000], t[k:k + 50_000])
        host = _export_all(wc)
        dev, dsrc = wc.export(np.float64, with_timestamps=True, with_source_index=True, device=True)
        torch.cuda.synchronize()
        assert dev.cpu().numpy().tobytes() == host[0].tobytes()
        assert dsrc.cpu().numpy().astype(np.uint64).tobytes() == host[1].tobytes()
        outs.append(host[0].tobytes() + host[1].tobytes())
        wc.close()
    assert outs[0] == outs[1]
