"""Scans in device memory (cticp_odometry_register_device, torch CUDA tensors) and point vectors written to device memory
(cticp_odometry_write_points_device, points_device) give exactly what the host paths give on the same values: summaries
(wall-clock fields aside), trajectories, the three point vectors and the map, byte for byte."""
import ctypes as C

import numpy as np
import pytest

import ct_icp_b200
from ct_icp_b200 import _abi as abi
from ct_icp_b200 import synthetic as syn

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

N_FRAMES = 7
WALL_CLOCK = ("odometry_total", "odometry_initialization", "odometry_try_register", "odometry_duration_sampling",
              "odometry_map_update", "odometry_transform")


@pytest.fixture(scope="module")
def seq():
    return syn.make_sequence(N_FRAMES + 1, syn.SMALL16, seed=1234)


def _options(eng, profile):
    if profile == "default_driving_ceres":
        o = eng.profile("default_driving")
        o.ct_icp_options.solver = abi.SOLVER["CERES"]
    elif profile == "robust_driving":
        o = eng.profile("robust_driving")
    else:   # the bench's GN options (BASELINE.json configs[1])
        o = eng.default_odometry_options()
        o.ct_icp_options.solver = abi.SOLVER["GN"]
        o.ct_icp_options.num_iters_icp = 5
        o.ct_icp_options.min_number_neighbors = 10
        o.map_options = eng.legacy_map_options(1.0, 20, 0.1)
        o.voxel_size, o.sample_voxel_size, o.max_distance = 0.5, 1.5, 100.0
        o.init_num_frames = 3
        if profile == "constant_velocity":
            o.motion_compensation = abi.MOTION_COMPENSATION["CONSTANT_VELOCITY"]
        elif profile == "adaptive":
            o.sampling = abi.SAMPLING["ADAPTIVE"]
    o.debug_print = 0
    o.ct_icp_options.debug_print = 0
    return o


def _summary_bytes(sm):
    s = sm.copy()
    for f in WALL_CLOCK:
        setattr(s, f, 0.0)
    for f in ("duration_total", "duration_init", "avg_duration_iter", "avg_duration_neighborhood", "avg_duration_solve"):
        setattr(s.icp_summary, f, 0.0)
    return bytes(memoryview(s))


def _state(od):
    tr = od.Trajectory()
    return (b"".join(bytes(memoryview(f)) for f in tr),
            [od.points(w).tobytes() for w in (abi.POINTS_CORRECTED, abi.POINTS_ALL_CORRECTED, abi.POINTS_KEYPOINTS)],
            od.GetMapPointCloud().tobytes())


def _assert_same(od_host, od_dev, sums_host, sums_dev):
    assert len(sums_host) == len(sums_dev)
    for i, (a, b) in enumerate(zip(sums_host, sums_dev)):
        assert _summary_bytes(a) == _summary_bytes(b), i
    sh, sd = _state(od_host), _state(od_dev)
    assert sh[0] == sd[0]
    for w in range(3):
        assert sh[1][w] == sd[1][w], w
    assert sh[2] == sd[2]


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("profile", ["gn", "default_driving_ceres", "robust_driving", "constant_velocity", "adaptive",
                                     "summary_points_all"])
def test_float64_tensors_match_host_buffers(eng, seq, profile):
    od_h, od_d = eng.odometry(_options(eng, profile)), eng.odometry(_options(eng, profile))
    if profile == "summary_points_all":
        od_h.set_summary_points(7)
        od_d.set_summary_points(7)
    sh, sd = [], []
    for s in seq[:N_FRAMES]:
        sh.append(od_h.RegisterFrame(s["xyz"], s["t"], s["frame_idx"]))
        sd.append(od_d.RegisterFrame(_cuda(s["xyz"]), _cuda(s["t"]), s["frame_idx"]))
        if profile == "summary_points_all":
            # straight after the call, while the eager egress may still write the world coordinates on its own stream
            for which in (abi.POINTS_ALL_CORRECTED, abi.POINTS_KEYPOINTS, abi.POINTS_CORRECTED):
                out = od_d.points_device(which, world=True, with_timestamps=True)
                ref = np.zeros(len(out), dtype=[("x", "<f8"), ("y", "<f8"), ("z", "<f8"), ("t", "<f8")])
                assert od_h.write_points(which, ref, world=True) == len(out)
                assert out.cpu().numpy().tobytes() == ref.tobytes(), which
        assert od_d.last_timing().h2d_bytes < od_h.last_timing().h2d_bytes   # no scan bytes go up
    _assert_same(od_h, od_d, sh, sd)
    od_h.close(), od_d.close()


def _record_dtype(xdt, tdt, step, xoff, toff):
    return np.dtype({"names": ["x", "y", "z", "t"], "formats": [xdt, xdt, xdt, tdt],
                     "offsets": [xoff, xoff + np.dtype(xdt).itemsize, xoff + 2 * np.dtype(xdt).itemsize, toff],
                     "itemsize": step})


def _records(s, xdt, tdt, step, xoff, toff, t_base=0.0, t_scale=1e6):
    rec = np.zeros(len(s["xyz"]), dtype=_record_dtype(xdt, tdt, step, xoff, toff))
    rec["x"], rec["y"], rec["z"] = s["xyz"][:, 0], s["xyz"][:, 1], s["xyz"][:, 2]
    t = s["t"]
    rec["t"] = t if np.dtype(tdt).kind == "f" else np.round((t - t_base) * t_scale)   # integer (micro)seconds
    return rec


def test_float32_xyzi_read_in_place(eng, seq):
    """An (N, 4) float32 xyzi tensor is read in place; the host equivalent is RegisterCloud on the same float32 records."""
    od_h, od_d = eng.odometry(_options(eng, "gn")), eng.odometry(_options(eng, "gn"))
    sh, sd = [], []
    for s in seq[:N_FRAMES]:
        rec = _records(s, np.float32, np.float64, 24, 0, 16)
        sh.append(od_h.RegisterCloud(rec, s["frame_idx"]))
        xyzi = torch.zeros((len(rec), 4), dtype=torch.float32, device="cuda")
        xyzi[:, :3] = torch.from_numpy(np.stack([rec["x"], rec["y"], rec["z"]], axis=1)).cuda()
        xyzi[:, 3] = 7.0
        sd.append(od_d.RegisterFrame(xyzi, _cuda(rec["t"]), s["frame_idx"]))
    _assert_same(od_h, od_d, sh, sd)
    od_h.close(), od_d.close()


@pytest.mark.parametrize("tdt", [np.float64, np.float32, np.uint32, np.int32])
def test_packed_records_with_unaligned_fields(eng, seq, tdt):
    """PointCloud2-like records in a uint8 CUDA tensor: x at byte 1, t right behind z, nothing aligned."""
    od_h, od_d = eng.odometry(_options(eng, "gn")), eng.odometry(_options(eng, "gn"))
    step, xoff, toff = 13 + np.dtype(tdt).itemsize + 2, 1, 13
    code = abi.DTYPE[np.dtype(tdt).name]
    sh, sd = [], []
    for s in seq[:6]:
        rec = _records(s, np.float32, tdt, step, xoff, toff, t_base=float(seq[0]["t"].min()))
        sh.append(od_h.RegisterCloud(rec, s["frame_idx"]))
        buf = _cuda(rec.view(np.uint8))
        p = buf.data_ptr()
        scan = abi.DeviceScan(p + xoff, step, p + toff, step, len(rec), abi.DTYPE["float32"], code)
        sd.append(od_d.register_device(scan, s["frame_idx"], stream=torch.cuda.current_stream().cuda_stream))
    _assert_same(od_h, od_d, sh, sd)
    od_h.close(), od_d.close()


@pytest.mark.parametrize("tdt,toff,step", [(np.int8, 25, 27), (np.uint8, 25, 26), (np.int16, 25, 28),
                                           (np.uint16, 26, 28)])
def test_packed_float64_records_with_narrow_timestamps(eng, seq, tdt, toff, step):
    """float64 x, y, z at byte 1 (byte-assembled loads) with 1- and 2-byte timestamps, aligned and not: each frame's
    timestamps quantised to 255 (1-byte types) or 2000 (2-byte types) steps."""
    od_h, od_d = eng.odometry(_options(eng, "gn")), eng.odometry(_options(eng, "gn"))
    code = abi.DTYPE[np.dtype(tdt).name]
    info = np.iinfo(tdt)
    sh, sd = [], []
    for s in seq[:6]:
        t0, t1 = float(s["t"].min()), float(s["t"].max())
        xyz = s["xyz"] + 1e-9 * (np.arange(len(s["xyz"]))[:, None] % 4 == 0)   # with the residual plane
        lo, hi = max(info.min, -1000), min(info.max, 1000)
        rec = _records({"xyz": xyz, "t": s["t"]}, np.float64, tdt, step, 1, toff, t_scale=0.0)
        v = np.round((s["t"] - t0) * ((hi - lo - 1) / (t1 - t0)))
        rec["t"] = v + (lo + 1 if info.min < 0 else 0)
        sh.append(od_h.RegisterCloud(rec, s["frame_idx"]))
        buf = _cuda(rec.view(np.uint8))
        p = buf.data_ptr()
        scan = abi.DeviceScan(p + 1, step, p + toff, step, len(rec), abi.DTYPE["float64"], code)
        sd.append(od_d.register_device(scan, s["frame_idx"], stream=torch.cuda.current_stream().cuda_stream))
    _assert_same(od_h, od_d, sh, sd)
    od_h.close(), od_d.close()


def test_float64_coordinates_that_need_the_lo_plane(eng, seq):
    od_h, od_d = eng.odometry(_options(eng, "gn")), eng.odometry(_options(eng, "gn"))
    sh, sd = [], []
    for s in seq[:6]:
        xyz = s["xyz"] + 1e-9 * (np.arange(len(s["xyz"]))[:, None] % 3 == 0)
        assert np.any(xyz.astype(np.float32).astype(np.float64) != xyz)
        # timestamps as float32, any stride: every other element of a longer tensor
        t = s["t"].astype(np.float32)
        t2 = torch.zeros(2 * len(t), dtype=torch.float32, device="cuda")
        t2[::2] = _cuda(t)
        sh.append(od_h.RegisterFrame(xyz, t.astype(np.float64), s["frame_idx"]))
        sd.append(od_d.RegisterFrame(_cuda(xyz), t2[::2], s["frame_idx"]))
    _assert_same(od_h, od_d, sh, sd)
    od_h.close(), od_d.close()


def test_estimate_and_motion_prior(eng, seq):
    """RegisterFrameWithEstimate with estimate timestamps other than the scan's min / max, and a caller motion prior."""
    od_h, od_d = eng.odometry(_options(eng, "gn")), eng.odometry(_options(eng, "gn"))
    mm_opts = eng.default_odometry_options().default_motion_model
    sh, sd = [], []
    for i, s in enumerate(seq[:N_FRAMES]):
        if i < 2:
            sh.append(od_h.RegisterFrame(s["xyz"], s["t"], s["frame_idx"]))
            sd.append(od_d.RegisterFrame(_cuda(s["xyz"]), _cuda(s["t"]), s["frame_idx"]))
            continue
        prev = od_h.Trajectory()[-1]
        est = prev.copy()
        est.begin_pose = prev.end_pose.copy()
        est.begin_pose.dest_timestamp = float(s["t"].min()) - 0.004
        est.end_pose.dest_timestamp = float(s["t"].max()) + 0.007
        prior = abi.MotionPrior(mm_opts, prev) if i % 2 else None
        sh.append(od_h.RegisterFrameWithEstimate(s["xyz"], s["t"], est, s["frame_idx"], motion_model=prior))
        sd.append(od_d.RegisterFrameWithEstimate(_cuda(s["xyz"]), _cuda(s["t"]), est, s["frame_idx"], motion_model=prior))
    _assert_same(od_h, od_d, sh, sd)
    od_h.close(), od_d.close()


def test_producer_stream_order(eng, seq):
    """Each scan is written into the same device buffers by a copy on a side stream, behind a ~20 ms spin, just before a
    call that names that stream: the engine must read what the copy writes, not what the buffers held before."""
    od_h, od_d = eng.odometry(_options(eng, "gn")), eng.odometry(_options(eng, "gn"))
    cap = max(len(s["xyz"]) for s in seq)
    xyz_buf = torch.zeros((cap, 3), dtype=torch.float64, device="cuda")
    t_buf = torch.zeros(cap, dtype=torch.float64, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())   # the buffers' zero fill
    sh, sd = [], []
    for s in seq[:N_FRAMES]:
        n = len(s["xyz"])
        hx = torch.from_numpy(s["xyz"]).pin_memory()
        ht = torch.from_numpy(s["t"]).pin_memory()
        sh.append(od_h.RegisterFrame(s["xyz"], s["t"], s["frame_idx"]))
        with torch.cuda.stream(side):
            torch.cuda._sleep(40_000_000)
            xyz_buf[:n].copy_(hx, non_blocking=True)
            t_buf[:n].copy_(ht, non_blocking=True)
            sd.append(od_d.RegisterFrame(xyz_buf[:n], t_buf[:n], s["frame_idx"]))
    torch.cuda.synchronize()
    _assert_same(od_h, od_d, sh, sd)
    od_h.close(), od_d.close()


def test_errors_leave_the_sequence_equal_to_the_host_path(eng, seq):
    cap = max(len(s["xyz"]) for s in seq) + 16
    o = _options(eng, "gn")
    o.max_points_per_frame = cap
    od_h, od_d = eng.odometry(o), eng.odometry(o)
    sh, sd = [], []

    def both(host_call, dev_call):
        rh = rd = None
        try:
            sh.append(host_call())
        except ct_icp_b200.CticpError as e:
            rh = e.code
        try:
            sd.append(dev_call())
        except ct_icp_b200.CticpError as e:
            rd = e.code
        assert rh == rd
        return rd

    for i, s in enumerate(seq[:N_FRAMES]):
        xd, td = _cuda(s["xyz"]), _cuda(s["t"])
        if i == 2:
            # a host pointer to the C entry
            scan = abi.DeviceScan(s["xyz"].ctypes.data, 24, s["t"].ctypes.data, 8, len(s["t"]), 8, 8)
            with pytest.raises(ct_icp_b200.CticpError) as e:
                od_d.register_device(scan, s["frame_idx"])
            assert e.value.code == abi.ERR_INVALID_ARGUMENT
            # unknown dtypes
            for xdt, tdt in ((8, 9), (5, 8)):
                scan = abi.DeviceScan(xd.data_ptr(), 24, td.data_ptr(), 8, len(s["t"]), xdt, tdt)
                with pytest.raises(ct_icp_b200.CticpError) as e:
                    od_d.register_device(scan, s["frame_idx"])
                assert e.value.code == abi.ERR_INVALID_ARGUMENT
            # more points than max_points_per_frame (the buffers hold all of them)
            big_x, big_t = np.concatenate([s["xyz"]] * 2), np.concatenate([s["t"]] * 2)
            assert both(lambda: od_h.RegisterFrame(big_x, big_t, s["frame_idx"]),
                        lambda: od_d.RegisterFrame(_cuda(big_x), _cuda(big_t), s["frame_idx"])) == abi.ERR_CAPACITY
        if i == 4:
            # a timestamp outside the estimate's interval
            est = od_h.Trajectory()[-1].copy()
            est.begin_pose.dest_timestamp = float(s["t"].min()) + 0.01
            est.end_pose.dest_timestamp = float(s["t"].max())
            assert both(lambda: od_h.RegisterFrameWithEstimate(s["xyz"], s["t"], est, s["frame_idx"]),
                        lambda: od_d.RegisterFrameWithEstimate(xd, td, est, s["frame_idx"])) == abi.ERR_TIMESTAMP
        assert both(lambda: od_h.RegisterFrame(s["xyz"], s["t"], s["frame_idx"]),
                    lambda: od_d.RegisterFrame(xd, td, s["frame_idx"])) is None
    # a tensor on the host or of another dtype is refused before the C call
    with pytest.raises(ValueError):
        od_d.RegisterFrame(_cuda(seq[0]["xyz"]), torch.from_numpy(seq[0]["t"]), 0)
    with pytest.raises(ValueError):
        od_d.RegisterFrame(_cuda(seq[0]["xyz"]).to(torch.int32), _cuda(seq[0]["t"]), 0)
    _assert_same(od_h, od_d, sh, sd)
    od_h.close(), od_d.close()


SINKS = [  # (x dtype, t dtype or None, point_step, x offset, t offset, world)
    (np.float32, np.float64, 20, 0, 12, 1),
    (np.float64, np.float32, 37, 1, 29, 0),
    (np.float64, None, 40, 8, 0, 1),
]


@pytest.mark.parametrize("sink_idx", range(len(SINKS)))
def test_write_points_device_bytes_equal_write_points(eng, seq, sink_idx):
    xdt, tdt, step, xoff, toff, world = SINKS[sink_idx]
    od = eng.odometry(_options(eng, "gn"))
    for s in seq[:5]:
        xyz = s["xyz"] + 1e-9 * (np.arange(len(s["xyz"]))[:, None] % 5 == 0)   # with the residual plane
        od.RegisterFrame(_cuda(xyz), _cuda(s["t"]), s["frame_idx"])
    side = torch.cuda.Stream()
    for which in (abi.POINTS_CORRECTED, abi.POINTS_ALL_CORRECTED, abi.POINTS_KEYPOINTS):
        count = od.write_points_device(which, abi.CloudSink(None, 0, step, xoff, 0, 0, 0, world))
        assert count > 0
        for cap in (count, count - 5):
            n_rec = count + 3
            host = np.full(n_rec * step, 0xAB, dtype=np.uint8)
            dev = torch.full((n_rec * step,), 0xAB, dtype=torch.uint8, device="cuda")
            side.wait_stream(torch.cuda.current_stream())   # the fill: the engine writes after what `side` queued
            args = (cap, step, xoff, abi.DTYPE[np.dtype(xdt).name], toff,
                    abi.DTYPE[np.dtype(tdt).name] if tdt else 0, world)
            rh = od.b.fn("odometry_write_points")(od.h, which, C.byref(abi.CloudSink(host.ctypes.data, *args)))
            rd = od.write_points_device(which, abi.CloudSink(dev.data_ptr(), *args), side.cuda_stream)
            assert rh == rd == count
            with torch.cuda.stream(side):   # read on the stream the engine was told about
                got = dev.cpu().numpy()
            assert got.tobytes() == host.tobytes(), (which, cap)
    # points_device: the (n, 4) world + timestamp tensor equals write_points into the same layout
    for which in (abi.POINTS_CORRECTED, abi.POINTS_KEYPOINTS):
        ref = np.zeros(od.write_points_device(which, abi.CloudSink(None, 0, 0, 0, 0, 0, 0, 0)),
                       dtype=[("x", "<f8"), ("y", "<f8"), ("z", "<f8"), ("t", "<f8")])
        od.write_points(which, ref, world=True)
        out = od.points_device(which, world=True, dtype=torch.float64, with_timestamps=True)
        assert out.shape == (len(ref), 4)
        assert out.cpu().numpy().tobytes() == ref.tobytes()
    od.close()
