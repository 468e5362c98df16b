"""Continuous trajectories on the device (cticp_trajectory_*): poses and points against the CPU restatement of
slam::LinearContinuousTrajectory (tests/oracle_trajectory), every accepted record layout with host and device paths byte
for byte, a registered sequence against its own ALL_CORRECTED points, 64 concatenated scans, stream order, refusals."""
import ctypes as C

import numpy as np
import pytest

import ct_icp_b200
from ct_icp_b200 import _abi as abi
from conftest import get_sequence
from oracle_trajectory_lib import trajectory_oracle

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

T_DTYPES = ["int8", "uint8", "int16", "uint16", "int32", "uint32", "float32", "float64"]


@pytest.fixture(scope="module")
def tor():
    return trajectory_oracle()


def _pose(quat, tr, ts, fid, ref_fid=0, ref_ts=0.0):
    p = abi.Pose.make(quat=quat, tr=tr, dest_timestamp=ts, dest_frame_id=fid)
    p.ref_frame_id, p.ref_timestamp = ref_fid, ref_ts
    return p


def _quat(rng, spread=None, near=None):
    if near is None:
        q = rng.normal(size=4)
    else:
        q = np.asarray(near) + rng.normal(scale=spread, size=4)
    return q / np.linalg.norm(q)


def random_trajectory(rng, n, shape):
    """arbitrary: n poses, frames of 1-4 poses, any rotation between neighbours; odometry: n // 2 frames of begin / end
    poses with a small motion, boundaries equal to the next frame's begin timestamp half of the time"""
    poses = []
    if shape == "arbitrary":
        ts = np.sort(rng.uniform(-50.0, 50.0, n))
        fid = 0
        left = int(rng.integers(1, 5))
        for k in range(n):
            poses.append(_pose(_quat(rng), rng.uniform(-100, 100, 3), float(ts[k]), fid, 0, 1.5))
            left -= 1
            if left == 0:
                fid += int(rng.integers(1, 3))   # leaves some frame ids absent
                left = int(rng.integers(1, 5))
        return poses
    q = _quat(rng)
    tr = np.zeros(3)
    t = 100.0
    for k in range(max(n // 2, 1)):
        b = t
        e = b + 0.1
        fb = abi.Frame()
        q1 = _quat(rng, 0.02, q)
        tr1 = tr + rng.normal(scale=1.0, size=3)
        fb.begin_pose, fb.end_pose = _pose(q, tr, b, k), _pose(q1, tr1, e, k)
        poses += [fb.begin_pose, fb.end_pose]
        q, tr = q1, tr1
        t = e if rng.random() < 0.5 else e + 0.003
    return poses[:n] if n > 1 else poses[:1]


def queries(rng, P, m):
    """timestamps exactly at poses, between poses, between frames, below min, above max and NaN, with frame ids of
    frames present and absent (never above the last)"""
    ts = P["dest_timestamp"]
    fids = P["dest_frame_id"]
    k = rng.integers(0, len(ts), m)
    kind = rng.integers(0, 6, m)
    t = ts[k].copy()
    nxt = ts[np.minimum(k + 1, len(ts) - 1)]
    t = np.where(kind == 1, ts[k] + rng.random(m) * (nxt - ts[k]), t)
    t = np.where(kind == 2, ts[k] + 0.5 * (nxt - ts[k]), t)
    t = np.where(kind == 3, ts.min() - rng.uniform(0.001, 10, m), t)
    t = np.where(kind == 4, ts.max() + rng.uniform(0.001, 10, m), t)
    t = np.where(kind == 5, np.nan, t)
    f = fids[k].astype(np.int64) + rng.integers(-1, 2, m)
    f = np.clip(f, 0, int(fids.max())).astype(np.uint32)
    return t, f


def assert_poses_match(a, b):
    """ids and timestamps identical (the lerp of the timestamps rounds as the host's), rotations to 1e-14, translations
    to 1e-12 m; a pose the lookup returns unchanged is identical byte for byte"""
    for name in ("ref_frame_id", "dest_frame_id", "ref_timestamp", "dest_timestamp"):
        np.testing.assert_array_equal(a[name], b[name], err_msg=name)
    np.testing.assert_allclose(a["quat"], b["quat"], rtol=0, atol=1e-14)
    np.testing.assert_allclose(a["tr"], b["tr"], rtol=0, atol=1e-12)


@pytest.mark.parametrize("shape", ["arbitrary", "odometry"])
@pytest.mark.parametrize("n", [1, 2, 3, 17, 256, 5000])
def test_poses_and_points_against_the_oracle(eng, tor, shape, n):
    rng = np.random.default_rng(1000 * n + (shape == "odometry"))
    poses = random_trajectory(rng, n, shape)
    te, to = eng.continuous_trajectory(poses), tor.continuous_trajectory(poses)
    P = te.poses()
    assert P.tobytes() == to.poses().tobytes()
    t, f = queries(rng, P, 4000)
    for fid in (None, f):
        ge, go = te.interpolate(t, fid), to.interpolate(t, fid)
        assert_poses_match(ge, go)
        if fid is None:   # below the minimum, above the maximum, NaN: equal lookup indices, the pose itself
            same = np.isnan(t) | (t < P["dest_timestamp"].min()) | (t > P["dest_timestamp"].max())
            assert same.any() and ge[same].tobytes() == go[same].tobytes()
    xyz = rng.uniform(-200.0, 200.0, (len(t), 3)) / np.sqrt(3)
    for segs in (None, "frames"):
        seg = None
        tt = t
        if segs:
            order = np.argsort(f, kind="stable")
            fs, tt, xyz_s = f[order], t[order], xyz[order]
            ids, starts = np.unique(fs, return_index=True)
            seg = (np.append(starts[1:], len(fs)), ids)
        else:
            xyz_s = xyz
        we = te.transform(xyz_s, tt, seg, with_timestamps=True)
        wo = to.transform(xyz_s, tt, seg, with_timestamps=True)
        np.testing.assert_allclose(we[:, :3], wo[:, :3], rtol=0, atol=1e-10)
        assert we[:, 3].tobytes() == wo[:, 3].tobytes()


def _records(rng, n, xdt, tdt, pad_front, t0=100.0, t1=100.5):
    """packed records: pad bytes, x, y, z, one pad byte, t — misaligned for every scalar wider than a byte"""
    dt = np.dtype([("pad", "u1", (pad_front,)), ("x", xdt), ("y", xdt), ("z", xdt), ("gap", "u1"), ("t", tdt)]) \
        if pad_front else np.dtype([("x", xdt), ("y", xdt), ("z", xdt), ("gap", "u1"), ("t", tdt)])
    rec = np.zeros(n, dtype=dt)
    for c in "xyz":
        rec[c] = rng.uniform(-80, 80, n)
    if np.dtype(tdt).kind == "f":
        rec["t"] = rng.uniform(t0, t1, n)
    else:
        info = np.iinfo(tdt)
        rec["t"] = rng.integers(max(info.min, -100), min(info.max, 200), n)
    return rec


def _device_scan(dev_bytes, rec):
    f = rec.dtype.fields
    base = dev_bytes.data_ptr()
    return abi.DeviceScan(base + f["x"][1], rec.dtype.itemsize, base + f["t"][1], rec.dtype.itemsize, len(rec),
                          abi.DTYPE[f["x"][0].name], abi.DTYPE[f["t"][0].name])


def _sink_dtype(odt, with_t, lead=3):
    fields = [("lead", "u1", (lead,)), ("x", odt), ("y", odt), ("z", odt)]
    if with_t:
        fields.append(("t", odt))
    fields.append(("tail", "u1", (2,)))
    return np.dtype(fields)


@pytest.mark.parametrize("xdt", ["float32", "float64"])
@pytest.mark.parametrize("tdt", T_DTYPES)
def test_every_input_layout_host_and_device_byte_identical(eng, tor, xdt, tdt):
    rng = np.random.default_rng(2 * T_DTYPES.index(tdt) + (xdt == "float64"))
    lo_t, hi_t = (-100.0, 200.0) if np.dtype(tdt).kind in "iu" else (100.0, 100.5)
    if np.dtype(tdt).kind == "u" or tdt == "int8":
        lo_t = 0.0 if np.dtype(tdt).kind == "u" else -100.0
        hi_t = 120.0
    poses = [_pose(_quat(rng), rng.uniform(-10, 10, 3), float(ts), k // 2)
             for k, ts in enumerate(np.linspace(lo_t, hi_t, 8))]
    te, to = eng.continuous_trajectory(poses), tor.continuous_trajectory(poses)
    n = 3001
    for pad in (0, 1):
        rec = _records(rng, n, xdt, tdt, pad, lo_t, hi_t)
        dev_rec = torch.from_numpy(rec.view(np.uint8).copy()).cuda()
        scan = _device_scan(dev_rec, rec)
        for odt in ("float32", "float64"):
            for with_t in (False, True):
                sdt = _sink_dtype(odt, with_t)
                for cap in (n, n - 7, 0):
                    host = np.full((n + 2) * sdt.itemsize, 0xAB, dtype=np.uint8).view(sdt)
                    dev = torch.full((len(host) * sdt.itemsize,), 0xAB, dtype=torch.uint8, device="cuda")
                    f = sdt.fields
                    args = (cap, sdt.itemsize, f["x"][1], abi.DTYPE[odt], f["t"][1] if with_t else 0,
                            abi.DTYPE[odt] if with_t else 0, 1)
                    rh = te.b.fn("trajectory_transform")(te.h, C.byref(Odometry_view(rec)), None, None, 0,
                                                        C.byref(abi.CloudSink(host.ctypes.data, *args)))
                    rd = te.transform_device(scan, abi.CloudSink(dev.data_ptr(), *args),
                                             stream=torch.cuda.current_stream().cuda_stream)
                    assert rh == rd == n
                    got = dev.cpu().numpy()
                    assert got.tobytes() == host.view(np.uint8).tobytes(), (pad, odt, with_t, cap)
                    assert (got[cap * sdt.itemsize:] == 0xAB).all()
                    if cap == n:
                        ref = np.full((n + 2) * sdt.itemsize, 0xAB, dtype=np.uint8).view(sdt)
                        to.transform_records(rec, ref)
                        for c in "xyz":
                            np.testing.assert_allclose(host[c][:n], ref[c][:n], rtol=0,
                                                       atol=1e-10 if odt == "float64" else 2e-5)
                        if with_t:
                            assert host["t"][:n].tobytes() == ref["t"][:n].tobytes()
                            np.testing.assert_array_equal(host["t"][:n], rec["t"].astype(odt))


def Odometry_view(rec):
    from ct_icp_b200._binding import Odometry
    return Odometry._cloud_view(rec)


def test_tensor_and_numpy_paths(eng):
    rng = np.random.default_rng(2)
    poses = random_trajectory(rng, 40, "odometry")
    te = eng.continuous_trajectory(poses)
    P = te.poses()
    n = 10000
    xyz = rng.uniform(-50, 50, (n, 4)).astype(np.float32)
    t = rng.uniform(P["dest_timestamp"][0], P["dest_timestamp"][-1], n)
    for dtype in (np.float32, np.float64):
        a = te.transform(xyz[:, :3], t, dtype=dtype, with_timestamps=True)
        b = te.transform(torch.from_numpy(xyz).cuda(), torch.from_numpy(t).cuda(), dtype=dtype, with_timestamps=True)
        assert b.cpu().numpy().tobytes() == np.ascontiguousarray(a).tobytes()


def _options(eng):
    o = eng.default_odometry_options()
    o.ct_icp_options.solver = abi.SOLVER["GN"]
    o.ct_icp_options.min_number_neighbors = 10
    o.map_options = eng.legacy_map_options(1.0, 20, 0.1)
    o.init_num_frames = 3
    o.debug_print = 0
    o.ct_icp_options.debug_print = 0
    return o


def test_against_a_registered_sequence(eng):
    """Each frame's scan, transformed as its own segment along the trajectory of Odometry.Trajectory(), lands on that
    frame's ALL_CORRECTED world points (those use the fp32 alpha of the registration, this path does not)"""
    seq = get_sequence("small16", 8)
    od = eng.odometry(_options(eng))
    expected = []
    for s in seq:
        sm = od.RegisterFrame(s["xyz"], s["t"], s["frame_idx"])
        assert sm.success, sm.error_message
        expected.append(od.all_corrected_points())
    traj = eng.continuous_trajectory(od.Trajectory())
    xyz = np.concatenate([s["xyz"] for s in seq])
    t = np.concatenate([s["t"] for s in seq])
    ends = np.cumsum([len(s["xyz"]) for s in seq])
    fids = [s["frame_idx"] for s in seq]
    w = traj.transform(xyz, t, segments=(ends, fids))
    wd = traj.transform(torch.from_numpy(xyz).cuda(), torch.from_numpy(t).cuda(), segments=(ends, fids)).cpu().numpy()
    assert wd.tobytes() == w.tobytes()
    ref = np.concatenate([e["world"] for e in expected])
    assert np.abs(w - ref).max() <= 1e-5, np.abs(w - ref).max()
    od.close()


def test_64_concatenated_scans(eng, tor):
    """64 bench-size scans (~130k points each) device to device, every 997th point against the oracle"""
    rng = np.random.default_rng(64)
    poses = random_trajectory(rng, 128, "odometry")
    te, to = eng.continuous_trajectory(poses), tor.continuous_trajectory(poses)
    P = te.poses()
    per = 130000
    n = 64 * per
    g = torch.Generator(device="cuda").manual_seed(5)
    xyz = (torch.rand((n, 4), generator=g, device="cuda", dtype=torch.float32) - 0.5) * 200.0
    fr = torch.arange(n, device="cuda") // per
    b = torch.from_numpy(P["dest_timestamp"][0::2].copy()).cuda()
    e = torch.from_numpy(P["dest_timestamp"][1::2].copy()).cuda()
    t = b[fr] + torch.rand(n, generator=g, device="cuda", dtype=torch.float64) * (e[fr] - b[fr])
    ends = np.arange(1, 65, dtype=np.uint64) * per
    fids = np.arange(64, dtype=np.uint32)
    out = te.transform(xyz, t, segments=(ends, fids), dtype=np.float64)
    torch.cuda.synchronize()
    idx = np.arange(0, n, 997)
    xs = xyz[idx].cpu().numpy().astype(np.float64)
    ts = t[idx].cpu().numpy()
    seg_of = idx // per
    got = out[idx].cpu().numpy()
    ref = np.empty_like(got)
    for s in np.unique(seg_of):
        m = seg_of == s
        ref[m] = to.transform(xs[m], ts[m], segments=(np.array([m.sum()]), np.array([s])))
    np.testing.assert_allclose(got, ref, rtol=0, atol=1e-10)
    # the same by timestamp (the frames do not overlap in time)
    out_t = te.transform(xyz, t, dtype=np.float64)
    ref_t = to.transform(xs, ts)
    np.testing.assert_allclose(out_t[idx].cpu().numpy(), ref_t, rtol=0, atol=1e-10)


def test_producer_and_consumer_stream_order(eng):
    """the records are written on a side stream behind a ~20 ms spin just before the call that names it, and the sink
    is read on that stream: the engine reads what the copy wrote and the reader sees what the engine wrote"""
    rng = np.random.default_rng(9)
    poses = random_trajectory(rng, 10, "odometry")
    te = eng.continuous_trajectory(poses)
    P = te.poses()
    n = 50000
    xyz_buf = torch.zeros((n, 3), dtype=torch.float64, device="cuda")
    t_buf = torch.zeros(n, dtype=torch.float64, device="cuda")
    out = torch.zeros((n, 3), dtype=torch.float64, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    for k in range(3):
        xyz = rng.uniform(-30, 30, (n, 3))
        t = rng.uniform(P["dest_timestamp"][0], P["dest_timestamp"][-1], n)
        expected = te.transform(xyz, t)
        hx, ht = torch.from_numpy(xyz).pin_memory(), torch.from_numpy(t).pin_memory()
        with torch.cuda.stream(side):
            torch.cuda._sleep(40_000_000)
            xyz_buf.copy_(hx, non_blocking=True)
            t_buf.copy_(ht, non_blocking=True)
            scan = abi.DeviceScan(xyz_buf.data_ptr(), 24, t_buf.data_ptr(), 8, n, abi.DTYPE["float64"], abi.DTYPE["float64"])
            sink = abi.CloudSink(out.data_ptr(), n, 24, 0, abi.DTYPE["float64"], 0, 0, 1)
            assert te.transform_device(scan, sink, stream=side.cuda_stream) == n
            got = out.cpu().numpy()   # on the stream the engine was told about
        assert got.tobytes() == expected.tobytes(), k
    torch.cuda.synchronize()


def test_refusals_write_nothing(eng):
    rng = np.random.default_rng(4)
    poses = [_pose(_quat(rng), rng.uniform(-1, 1, 3), float(k), k // 2) for k in range(6)]   # frames 0, 1, 2
    te = eng.continuous_trajectory(poses)
    n = 1000
    xyz = torch.from_numpy(rng.uniform(-5, 5, (n, 3))).cuda()
    t = torch.from_numpy(rng.uniform(0, 5, n)).cuda()
    out = torch.full((n, 3), 7.0, dtype=torch.float64, device="cuda")
    good_scan = abi.DeviceScan(xyz.data_ptr(), 24, t.data_ptr(), 8, n, 8, 8)
    good_sink = abi.CloudSink(out.data_ptr(), n, 24, 0, 8, 0, 0, 1)
    host_xyz = np.zeros((n, 3))
    F = te.b.fn("trajectory_transform_device")

    def refused(scan, sink, ends=None, fids=None, ns=0):
        e = ends.ctypes.data if ends is not None else None
        f = fids.ctypes.data if fids is not None else None
        rc = F(te.h, C.byref(scan) if scan is not None else None, e, f, ns, C.byref(sink) if sink is not None else None,
               None)
        assert rc == abi.ERR_INVALID_ARGUMENT, rc
        torch.cuda.synchronize()
        assert bool((out == 7.0).all())

    def scan_with(**kw):
        s = good_scan.copy()
        for k, v in kw.items():
            setattr(s, k, v)
        return s

    def sink_with(**kw):
        s = good_sink.copy()
        for k, v in kw.items():
            setattr(s, k, v)
        return s

    refused(None, good_sink)
    refused(good_scan, None)
    refused(scan_with(xyz=None), good_sink)
    refused(scan_with(xyz_dtype=5), good_sink)
    refused(scan_with(t_dtype=9), good_sink)
    refused(good_scan, sink_with(xyz_dtype=6))
    refused(good_scan, sink_with(t_dtype=5, t_offset=0))
    refused(good_scan, sink_with(xyz_offset=4))              # x, y, z past point_step
    refused(good_scan, sink_with(t_dtype=8, t_offset=20))    # t past point_step
    refused(good_scan, sink_with(world=0))
    refused(scan_with(xyz=host_xyz.ctypes.data), good_sink)  # host memory: checked before any launch
    refused(good_scan, sink_with(data=host_xyz.ctypes.data))
    # described buffers that end 8 bytes past their allocation (the caching allocator's segment that holds the tensor)
    def segment_end(ptr):
        seg = next(g for g in torch.cuda.memory_snapshot() if g["address"] <= ptr < g["address"] + g["total_size"])
        return seg["address"] + seg["total_size"]

    near_end = segment_end(xyz.data_ptr()) - 10 * 24 + 8
    refused(scan_with(xyz=near_end, num_points=10), sink_with(capacity_points=10))
    near_end = segment_end(out.data_ptr()) - 10 * 24 + 8
    refused(scan_with(num_points=10), sink_with(data=near_end, capacity_points=10))
    u64, u32 = np.uint64, np.uint32
    refused(good_scan, good_sink, np.array([600, 500, n], u64), np.array([0, 1, 2], u32), 3)   # decreasing ends
    refused(good_scan, good_sink, np.array([500, n - 1], u64), np.array([0, 1], u32), 2)       # last end != n
    refused(good_scan, good_sink, np.array([500, n], u64), np.array([0, 3], u32), 2)           # frame beyond
    refused(good_scan, good_sink, None, np.array([0], u32), 1)                                  # null ends
    # the host variant refuses the same
    rec = np.zeros(n, dtype=[("x", "<f8"), ("y", "<f8"), ("z", "<f8"), ("t", "<f8")])
    sink_h = np.full(n, 7.0, dtype=[("x", "<f8"), ("y", "<f8"), ("z", "<f8")])
    with pytest.raises(ct_icp_b200.CticpError) as e:
        te.transform_records(rec, sink_h, segments=(np.array([n]), np.array([9])))
    assert e.value.code == abi.ERR_INVALID_ARGUMENT
    assert (sink_h.view(np.float64) == 7.0).all()
    with pytest.raises(ct_icp_b200.CticpError) as e:
        te.interpolate([2.5], [9])
    assert e.value.code == abi.ERR_INVALID_ARGUMENT
    # the refused calls left the trajectory usable
    assert te.transform_device(good_scan, good_sink) == n
    torch.cuda.synchronize()
    assert not bool((out == 7.0).any())
