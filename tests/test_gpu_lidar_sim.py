"""Spinning-LiDAR sweeps on the device (include/cticp.h, "Spinning-LiDAR sweeps") against the host caster tools/raycast.c
and the NumPy restatement of tests/lidar_sim_ref.py: ranges bit for bit (porous returns within 4 ulp), sweeps of three
sensors, batch independence, host and device sinks, the noise, registration of device sweeps against the oracle, and
the refusals."""
import numpy as np
import pytest

from conftest import frame_diff
from ct_icp_b200 import _abi as abi
from ct_icp_b200 import synthetic as syn
from ct_icp_b200._binding import CticpError
import lidar_sim_ref as ref
from test_gpu_parity import POSE_TOL_M, POSE_TOL_RAD, _sequence_options

pytestmark = pytest.mark.gpu


def _ulps(a, b):
    """|a - b| in units of the last place of b (0 where both are equal, inf included)"""
    same = (a == b) | (np.isnan(a) & np.isnan(b))
    fa, fb = np.where(np.isfinite(a), a, 0.0), np.where(np.isfinite(b), b, 1.0)
    d = np.abs(fa - fb) / np.spacing(np.abs(fb))
    return np.where(same, 0.0, np.where(np.isfinite(a) & np.isfinite(b), d, np.inf))


def _random_scene(rng, nb=300, nc=80, spread=60.0):
    lo = rng.uniform([-spread, -spread, 0.0], [spread, spread, 3.0], (nb, 3))
    boxes = np.concatenate([lo, lo + rng.uniform([0.2, 0.2, 0.3], [12.0, 12.0, 15.0], (nb, 3)), np.zeros((nb, 1))], 1)
    boxes[::3, 6] = rng.uniform(0.3, 3.0, len(boxes[::3]))   # porous
    cyl = np.concatenate([rng.uniform(-spread, spread, (nc, 2)), rng.uniform(0.05, 1.5, (nc, 1)),
                          rng.uniform(0.5, 12.0, (nc, 1))], 1)
    return boxes, cyl


def _hand_rays(boxes, cyl, R):
    """axis-parallel, vertical, box-corner and cylinder-tangent rays, rays from inside boxes, beyond the x-window and
    at boxes beyond max_range but inside the window"""
    o, d = [], []
    axes = [(1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)]
    for b in boxes[:40]:
        c = (b[:3] + b[3:6]) / 2
        for a in axes:   # from inside the box, and from outside along each axis toward it
            o.append(c), d.append(a)
            o.append(c - 30 * np.array(a, dtype=float)), d.append(a)
        for corner in ((b[0], b[1], b[5]), (b[3], b[4], b[2]), (b[0], b[4], b[5])):
            src = np.array([b[0] - 7.0, b[1] - 5.0, 1.7])
            v = np.array(corner) - src
            o.append(src), d.append(v / np.linalg.norm(v))
        o.append([b[3] + R + 5.0, (b[1] + b[4]) / 2, 1.0]), d.append((-1, 0, 0))   # outside the x-window
        o.append([(b[0] + b[3]) / 2, b[1] - 1.5 * R, 1.0]), d.append((0, 1, 0))     # beyond max_range, inside the window
    for cx, cy, r, h in cyl[:40]:
        src = np.array([cx - 10.0, cy - 3.0, 1.0])
        p = np.array([cx, cy]) - src[:2]
        L = np.linalg.norm(p)
        ang = np.arcsin(min(1.0, r / L))
        base = np.arctan2(p[1], p[0])
        for s in (-1, 1):   # the two silhouettes, slightly upward
            a = base + s * ang
            v = np.array([np.cos(a), np.sin(a), 0.05])
            o.append(src), d.append(v / np.linalg.norm(v))
        o.append([cx, cy, h + 2.0]), d.append((0, 0, -1))   # straight down onto the top
    return np.array(o, dtype=float), np.array(d, dtype=float)


def _random_rays(rng, n, spread=60.0):
    o = rng.uniform([-spread, -spread, 0.2], [spread, spread, 4.0], (n, 3))
    d = rng.normal(size=(n, 3))
    d[: n // 4, 2] = -np.abs(d[: n // 4, 2]) * 0.1
    return o, d / np.linalg.norm(d, axis=1)[:, None]


@pytest.mark.parametrize("seed", [1, 2])
def test_raycast_matches_the_host_caster(eng, seed):
    import torch
    rng = np.random.default_rng(seed)
    boxes, cyl = _random_scene(rng)
    R = 40.0
    o, d = _random_rays(rng, 200000)
    ho, hd = _hand_rays(boxes, cyl, R)
    o, d = np.concatenate([o, ho]), np.concatenate([d, hd])
    key = 0x9E3779B97F4A7C15 + seed
    solid = boxes.copy()
    solid[:, 6] = 0.0
    for bx, porous in ((solid, False), (boxes, True)):
        sc = eng.lidar_scene(bx, cyl)
        got = sc.raycast(o, d, R, key)
        want = ref.raycast(bx, cyl, o, d, R, key)
        assert np.array_equal(np.isfinite(got), np.isfinite(want))
        if porous:
            assert _ulps(got, want).max() <= 4
        else:
            assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
        assert (np.isfinite(want) & (want > R)).any()   # hits beyond max_range inside the window are kept
        dev = sc.raycast(torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda(), R, key)
        assert dev.cpu().numpy().tobytes() == got.tobytes()
    # without the ground plane: rays that do not descend are the host caster's; the others are no nearer than with it
    ng = eng.lidar_scene(solid, cyl, ground=False).raycast(o, d, R, key)
    wg = ref.raycast(solid, cyl, o, d, R, key)
    up = d[:, 2] >= 0
    assert np.array_equal(ng[up].view(np.uint64), wg[up].view(np.uint64))
    t_ground = np.where(d[:, 2] < 0, -o[:, 2] / np.where(d[:, 2] < 0, d[:, 2], -1.0), np.inf)
    nearer = ~up & (wg < t_ground)
    assert np.array_equal(ng[nearer].view(np.uint64), wg[nearer].view(np.uint64))
    assert (ng[~up] >= wg[~up]).all()
    assert np.isnan(eng.lidar_scene(solid, cyl).raycast(torch.tensor([[np.nan, 0, 1.0]]).double().cuda(),
                                                         torch.tensor([[1.0, 0, 0]]).double().cuda(), R).item())


@pytest.mark.parametrize("profile", ["street", "suburb"])
def test_urban_scene_hdl64e_rays_hit_and_miss_as_the_host_caster(eng, profile):
    scene = syn.UrbanScene(1234, profile=profile)
    traj = syn.Trajectory(height=syn.HDL64E.height)
    sc = eng.lidar_scene(scene.boxes, scene.cyl)
    ds = ref.sensor_directions(syn.HDL64E)
    for frame in (0, 40):
        t0 = frame * syn.HDL64E.period
        from scipy.spatial.transform import Rotation
        tc = ref.column_times(t0, syn.HDL64E)
        q = Rotation.from_matrix(traj.rotation(tc)).as_quat()
        j = np.tile(np.arange(syn.HDL64E.n_azimuth), syn.HDL64E.n_rings)
        o = traj.position(tc)[j]
        d = ref.qrot(ref.qnormalized(q)[j], ds)
        key = scene.seed * 1000003 + frame
        got = sc.raycast(o, d, syn.HDL64E.max_range, key)
        want = scene.raycast(o, d, syn.HDL64E.max_range, ray_seed=frame)
        assert np.array_equal(np.isfinite(got), np.isfinite(want)), profile
        assert _ulps(got, want).max() <= 4
        print("%s frame %d: %d hits of %d rays" % (profile, frame, int(np.isfinite(got).sum()), len(got)))


def _suburb():
    scene = syn.UrbanScene(1234, profile="suburb")
    return scene, syn.Trajectory(height=1.73)


@pytest.mark.parametrize("sensor", [syn.SMALL16, syn.HDL64, syn.DENSE128], ids=lambda s: s.name)
def test_sweeps_match_the_restatement(eng, sensor):
    scene, traj = _suburb()
    sc = eng.lidar_scene(scene.boxes, scene.cyl)
    tr = eng.continuous_trajectory(ref.trajectory_poses(traj, 2.0))
    frames = [(0.3, 3), (1.1, 11)]
    seed = 77
    raw = sc.sweeps(tr, sensor, frames, seed=seed, world=False, device=False)
    world = sc.sweeps(tr, sensor, frames, seed=seed, world=True, device=False)
    ends = np.concatenate([[0], raw["frame_ends"]]).astype(np.int64)
    assert np.array_equal(raw["frame_ends"], world["frame_ends"])
    for k, (t0, fid) in enumerate(frames):
        quat, trn = ref.device_columns(tr, sensor, t0)
        want = ref.sweep(scene.boxes, scene.cyl, sensor, t0, fid, seed, quat, trn)
        sl = slice(ends[k], ends[k + 1])
        assert np.array_equal(raw["ray_index"][sl], want["ray_index"]), (sensor.name, k)
        assert np.array_equal(raw["t"][sl].view(np.uint64), want["t"].view(np.uint64))
        # the ranges themselves, through the device caster on the restatement's rays
        got_r = sc.raycast(want["o"], want["dw"], sensor.max_range, (seed * 1000003 + fid) & (2 ** 64 - 1))
        assert np.array_equal(np.isfinite(got_r), np.isfinite(want["all_r"])) and _ulps(got_r, want["all_r"]).max() <= 4
        assert np.abs(raw["xyz"][sl] - want["raw"]).max() <= 1e-12
        assert np.abs(world["xyz"][sl] - want["world"]).max() <= 1e-12
        print("%s frame %d: %d points" % (sensor.name, fid, len(want["ray_index"])))


def test_frame_alone_equals_frame_in_batch_and_seeds(eng):
    import torch
    scene, traj = _suburb()
    sc = eng.lidar_scene(scene.boxes, scene.cyl)
    tr = eng.continuous_trajectory(ref.trajectory_poses(traj, 2.0))
    sensor = syn.SensorModel("noisy", 16, 15.0, -15.0, 900, 0.1, 1.0, 60.0, 1.5)
    sensor.noise_sigma = 0.03
    frames = [(0.1 * k, k) for k in range(12)]
    batch = sc.sweeps(tr, sensor, frames, seed=5)
    ends = np.concatenate([[0], batch["frame_ends"].cpu().numpy()]).astype(np.int64)
    for k in (0, 5, 11):
        one = sc.sweeps(tr, sensor, [frames[k]], seed=5)
        sl = slice(ends[k], ends[k + 1])
        for f in ("xyz", "t", "ray_index"):
            assert one[f].cpu().numpy().tobytes() == batch[f][sl].cpu().numpy().tobytes(), (k, f)
    again = sc.sweeps(tr, sensor, frames, seed=5)
    assert torch.equal(again["xyz"], batch["xyz"]) and torch.equal(again["ray_index"], batch["ray_index"])
    other = sc.sweeps(tr, sensor, frames, seed=6)
    n = min(len(other["t"]), len(batch["t"]))
    assert not torch.equal(other["xyz"][:n], batch["xyz"][:n])


@pytest.mark.parametrize("fmt,step,xoff,toff,tfmt", [("float64", 32, 0, 24, "float64"), ("float32", 16, 0, 12, "float32"),
                                                     ("float64", 41, 1, 29, "float64"), ("float32", 23, 3, 15, "float64")])
def test_host_and_device_sinks_write_the_same_bytes(eng, fmt, step, xoff, toff, tfmt):
    import torch
    scene, traj = _suburb()
    sc = eng.lidar_scene(scene.boxes, scene.cyl)
    tr = eng.continuous_trajectory(ref.trajectory_poses(traj, 2.0))
    sensor = syn.SMALL16
    frames = [(0.1 * k, 2 * k + 1) for k in range(6)]
    rng = np.random.default_rng(3)
    for world in (0, 1):
        n = int(sc.sweeps(tr, sensor, frames, seed=9, device=False)["frame_ends"][-1])
        fill = rng.integers(0, 256, n * step + 8, dtype=np.uint8)   # bytes outside the fields stay the caller's
        host = fill.copy()
        idx_h = np.zeros(n, dtype=np.uint32)
        ends_h = np.zeros(len(frames), dtype=np.uint64)
        sink = abi.CloudSink(host.ctypes.data, n, step, xoff, abi.DTYPE[fmt], toff, abi.DTYPE[tfmt], world)
        assert sc.sweeps_sink(tr, sensor, frames, 9, sink, idx_h, ends_h) == n
        dev = torch.from_numpy(fill.copy()).cuda()
        idx_d = torch.zeros(n, dtype=torch.int32, device="cuda")
        ends_d = torch.zeros(len(frames), dtype=torch.int64, device="cuda")
        dsink = abi.CloudSink(dev.data_ptr(), n, step, xoff, abi.DTYPE[fmt], toff, abi.DTYPE[tfmt], world)
        stream = torch.cuda.current_stream().cuda_stream
        sc.sweeps_device(tr, sensor, frames, 9, dsink, idx_d.data_ptr(), ends_d.data_ptr(), stream)
        assert dev.cpu().numpy().tobytes() == host.tobytes()
        assert idx_d.cpu().numpy().view(np.uint32).tobytes() == idx_h.tobytes()
        assert ends_d.cpu().numpy().view(np.uint64).tobytes() == ends_h.tobytes()
        cap = n // 3   # a short capacity writes that many records and still reports every frame's end
        host2 = fill.copy()
        sink2 = abi.CloudSink(host2.ctypes.data, cap, step, xoff, abi.DTYPE[fmt], toff, abi.DTYPE[tfmt], world)
        assert sc.sweeps_sink(tr, sensor, frames, 9, sink2, None, ends_h) == n
        assert host2[: cap * step].tobytes() == host[: cap * step].tobytes()
        assert host2[cap * step:].tobytes() == fill[cap * step:].tobytes()


def test_noise_statistics(eng):
    """~10^6 rays: the noise's mean and standard deviation agree with sigma within sampling error"""
    scene, traj = _suburb()
    sc = eng.lidar_scene(scene.boxes, scene.cyl)
    tr = eng.continuous_trajectory(ref.trajectory_poses(traj, 2.0))
    clean = syn.SensorModel(**{k: getattr(syn.HDL64E, k) for k in syn.SensorModel.__dataclass_fields__})
    noisy = syn.SensorModel(**{k: getattr(syn.HDL64E, k) for k in syn.SensorModel.__dataclass_fields__})
    noisy.noise_sigma = sigma = 0.05
    frames = [(0.1 * k, k) for k in range(8)]
    a = sc.sweeps(tr, clean, frames, seed=21)
    b = sc.sweeps(tr, noisy, frames, seed=21)
    ra, rb = a["xyz"].norm(dim=1).cpu().numpy(), b["xyz"].norm(dim=1).cpu().numpy()
    ia, ib = a["ray_index"].cpu().numpy(), b["ray_index"].cpu().numpy()
    fa = np.repeat(np.arange(8), np.diff(np.concatenate([[0], a["frame_ends"].cpu().numpy()])))
    fb = np.repeat(np.arange(8), np.diff(np.concatenate([[0], b["frame_ends"].cpu().numpy()])))
    ka = fa.astype(np.int64) << 32 | ia
    kb = fb.astype(np.int64) << 32 | ib
    common, xa, xb = np.intersect1d(ka, kb, return_indices=True)
    e = rb[xb] - ra[xa]
    inner = (ra[xa] > noisy.min_range + 6 * sigma) & (ra[xa] < noisy.max_range - 6 * sigma)
    e = e[inner]
    n = len(e)
    print("noise over %d rays: mean %.3e, std %.5f (sigma %.3f)" % (n, e.mean(), e.std(), sigma))
    assert n > 900000
    assert abs(e.mean()) < 5 * sigma / np.sqrt(n)
    assert abs(e.std() / sigma - 1.0) < 5 * np.sqrt(0.5 / n) + 1e-3
    again = sc.sweeps(tr, noisy, frames, seed=21)
    assert again["xyz"].cpu().numpy().tobytes() == b["xyz"].cpu().numpy().tobytes()


def test_device_sweeps_register_as_the_oracle(eng, orc):
    """HDL-64E sweeps generated into device memory and registered slice by slice with register_device, against the
    oracle's odometry on host copies. Gauss-Newton's hard gates can flip on a 1e-9 m difference; the policy of
    test_gpu_synthetic.py::test_courtyard_end_to_end_against_oracle_odometry applies: sampler counts identical on every
    frame, poses within 1e-4 m / 1e-4 rad up to the first flip of a residual count or map size."""
    import torch
    scene, traj = _suburb()
    sc = eng.lidar_scene(scene.boxes, scene.cyl)
    tr = eng.continuous_trajectory(ref.trajectory_poses(traj, 1.0))
    sensor = syn.SensorModel(**{k: getattr(syn.HDL64E, k) for k in syn.SensorModel.__dataclass_fields__})
    sensor.noise_sigma = 0.02
    m = 6
    out = sc.sweeps(tr, sensor, [(k * sensor.period, k) for k in range(m)], seed=1234)
    ends = out["frame_ends"].cpu().numpy().astype(np.int64)
    starts = np.concatenate([[0], ends[:-1]])
    rec = out["xyz"].stride(0) * out["xyz"].element_size()
    xyz_h, t_h = out["xyz"].cpu().numpy(), out["t"].cpu().numpy()
    stream = torch.cuda.current_stream().cuda_stream
    od_e, od_o = eng.odometry(_sequence_options(eng, "GN", init_num_frames=3)), \
        orc.odometry(_sequence_options(orc, "GN", init_num_frames=3))
    first_flip = None
    for k in range(m):
        a, n = int(starts[k]), int(ends[k] - starts[k])
        scan = abi.DeviceScan(out["xyz"].data_ptr() + a * rec, rec, out["t"].data_ptr() + a * rec, rec, n,
                              abi.DTYPE["float64"], abi.DTYPE["float64"])
        se = od_e.register_device(scan, k, stream=stream)
        so = od_o.RegisterFrame(np.ascontiguousarray(xyz_h[a:a + n]), np.ascontiguousarray(t_h[a:a + n]), k)
        assert se.success and so.success, (k, se.error_message, so.error_message)
        assert so.num_corrected_points == se.num_corrected_points and so.num_keypoints == se.num_keypoints, k
        if first_flip is None and (so.number_of_residuals != se.number_of_residuals or od_o.MapSize() != od_e.MapSize()):
            first_flip = k
        dt, dr = frame_diff(so.frame, se.frame, log=first_flip is None)
        if first_flip is None:
            assert dt < POSE_TOL_M and dr < POSE_TOL_RAD, (k, dt, dr)
        else:
            assert dt < 0.05 and dr < 5e-3, (k, dt, dr)   # two runs of the same chaotic iteration, not a tolerance claim
    print("HDL-64E device sweeps, %d frames: identical to the oracle up to frame %s" % (m, first_flip))
    assert first_flip is None or first_flip >= 3, first_flip


def test_refusals_write_nothing(eng):
    import torch
    scene, traj = _suburb()
    sc = eng.lidar_scene(scene.boxes[:50], scene.cyl[:10])
    tr = eng.continuous_trajectory(ref.trajectory_poses(traj, 1.0))
    host = np.full(64 * 32, 7, dtype=np.uint8)
    ends = np.full(3, 9, dtype=np.uint64)
    ok = [(0.0, 0)]

    def sink_of(buf, step=32, xdt="float64", tdt="float64"):
        return abi.CloudSink(buf.ctypes.data, 64, step, 0, abi.DTYPE.get(xdt, 99), 24, abi.DTYPE.get(tdt, 99), 0)

    def refused(code, sensor=syn.SMALL16, frames=ok, s=None):
        with pytest.raises(CticpError) as e:
            sc.sweeps_sink(tr, sensor, frames, 0, s or sink_of(host), None, ends)
        assert e.value.code == code
        assert (host == 7).all() and (ends == 9).all()

    refused(abi.ERR_INVALID_ARGUMENT, s=sink_of(host, xdt="int32"))
    refused(abi.ERR_INVALID_ARGUMENT, s=sink_of(host, tdt="int16"))
    refused(abi.ERR_INVALID_ARGUMENT, s=sink_of(host, step=16))
    refused(abi.ERR_INVALID_ARGUMENT, frames=[(float("nan"), 0)])
    bad = syn.SensorModel(**{k: getattr(syn.SMALL16, k) for k in syn.SensorModel.__dataclass_fields__})
    bad.noise_sigma = -1.0
    refused(abi.ERR_INVALID_ARGUMENT, sensor=bad)
    wide = syn.SensorModel("wide", 1 << 16, 10.0, -10.0, 1 << 16, 0.1, 1.0, 60.0, 1.5)
    refused(abi.ERR_CAPACITY, sensor=wide)
    for boxes, cyl in (([[0, 0, 0, -1, 1, 1, 0]], ()), ([[0, 0, 0, 1, 1, 1, -0.5]], ()), (([0, 0, 0, 1, np.inf, 1, 0],), ()),
                       ((), [[0, 0, -1.0, 2.0]])):
        with pytest.raises(CticpError) as e:
            eng.lidar_scene(boxes, cyl)
        assert e.value.code == abi.ERR_INVALID_ARGUMENT
    # device: host memory, a short buffer, misaligned frame ends / ray indices, a short ray-cast output
    rec = torch.full((64, 4), 7.0, dtype=torch.float64, device="cuda")
    ends_d = torch.full((4,), 9, dtype=torch.int64, device="cuda")
    idx_d = torch.full((70,), 9, dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    dsink = abi.CloudSink(rec.data_ptr(), 64, 32, 0, abi.DTYPE["float64"], 24, abi.DTYPE["float64"], 0)

    def segment_end(ptr):   # the caching allocator's segment that holds the tensor: the allocation the check sees
        seg = next(g for g in torch.cuda.memory_snapshot() if g["address"] <= ptr < g["address"] + g["total_size"])
        return seg["address"] + seg["total_size"]

    near_end = segment_end(rec.data_ptr()) - 10 * 32 + 8
    for s, i_ptr, e_ptr in ((sink_of(host), None, ends_d.data_ptr()),
                            (abi.CloudSink(near_end, 10, 32, 0, abi.DTYPE["float64"], 24, abi.DTYPE["float64"], 0), None,
                             ends_d.data_ptr()),
                            (dsink, None, ends.ctypes.data),
                            (dsink, None, ends_d.data_ptr() + 4),
                            (dsink, idx_d.data_ptr() + 2, ends_d.data_ptr())):
        with pytest.raises(CticpError) as e:
            sc.sweeps_device(tr, syn.SMALL16, ok, 0, s, i_ptr, e_ptr, stream)
        assert e.value.code == abi.ERR_INVALID_ARGUMENT
    o = torch.zeros((100, 3), dtype=torch.float64, device="cuda")
    out = torch.full((100,), 7.0, dtype=torch.float64, device="cuda")
    rc = eng.fn("lidar_scene_raycast_device")(sc.h, o.data_ptr(), o.data_ptr(), 100, 50.0, 0,
                                              segment_end(out.data_ptr()) - 8 * 50, None)   # 50 of 100 ranges fit
    assert rc == abi.ERR_INVALID_ARGUMENT
    torch.cuda.synchronize()
    assert (rec == 7.0).all() and (ends_d == 9).all() and (idx_d == 9).all() and (host == 7).all() and (ends == 9).all()
    assert (out == 7.0).all()
    with pytest.raises(CticpError) as e:
        sc.raycast(np.zeros((1, 3)), np.array([[np.nan, 0, 1.0]]), 10.0)
    assert e.value.code == abi.ERR_INVALID_ARGUMENT
    # a scene on a device that does not exist, or a trajectory on another device than the scene's
    if torch.cuda.device_count() > 1:
        tr1 = eng.continuous_trajectory(ref.trajectory_poses(traj, 1.0), device=1)
        with pytest.raises(CticpError) as e:
            sc.sweeps_sink(tr1, syn.SMALL16, ok, 0, sink_of(host), None, ends)
        assert e.value.code == abi.ERR_INVALID_ARGUMENT
    with pytest.raises(CticpError) as e:
        eng.lidar_scene(scene.boxes[:5], device=torch.cuda.device_count())
    assert e.value.code == abi.ERR_NO_DEVICE
    assert (host == 7).all() and (ends == 9).all()
