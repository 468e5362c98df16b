"""Dataset sequences on the device (include/cticp.h, "Dataset sequences") against the NumPy restatement of
tests/dataset_ref.py: NCLT velodyne_hits.bin streams packed from HDL-32 sweeps decoded bit for bit from host bytes,
device bytes and whole-frame chunks, skipping, the fallback walk, the refusals; the KITTI filter and the time ranges on
PLY records; and decoded frames registered with register_device against register_frame on the host copy."""
import numpy as np
import pytest

from ct_icp_b200 import _abi as abi
from ct_icp_b200 import synthetic as syn
from ct_icp_b200._binding import CticpError
import dataset_ref as ref
import lidar_sim_ref as lref
from test_gpu_parity import _sequence_options

pytestmark = pytest.mark.gpu


def _sweeps(eng, m, seed=3):
    scene, traj = syn.UrbanScene(1234, profile="suburb"), syn.Trajectory(height=1.0)
    sc = eng.lidar_scene(scene.boxes, scene.cyl)
    tr = eng.continuous_trajectory(lref.trajectory_poses(traj, m * 0.1 + 0.2))
    out = sc.sweeps(tr, syn.HDL32, [(k * syn.HDL32.period, k) for k in range(m)], seed=seed, device=False)
    return out, traj


def _pack(out, A, rng, empty_every=13):
    """each sweep split into A packets of random sizes (some empty), utime = the packet's first point's t in us"""
    ends = out["frame_ends"].astype(np.int64)
    starts = np.concatenate([[0], ends[:-1]])
    q = ref.quantise(out["xyz"])
    chunks = []
    for a, b in zip(starts, ends):
        cuts = np.sort(rng.integers(a, b + 1, A - 1))
        bounds = np.concatenate([[a], cuts, [b]])
        for k in range(A):
            lo, hi = bounds[k], bounds[k + 1]
            if k % empty_every == 5:
                hi = lo   # an empty packet; its points go to the next one
                if k + 1 < A:
                    bounds[k + 1] = lo
            ut = int(round(out["t"][lo] * 1e6)) if lo < len(out["t"]) else 0
            chunks.append(ref.pack_packet(1_300_000_000_000_000 + ut, q[lo:hi]))
    return chunks


@pytest.fixture(scope="module")
def stream_bytes(eng):
    rng = np.random.default_rng(11)
    out, _ = _sweeps(eng, 3)
    A = 40
    chunks = _pack(out, A, rng)
    chunks += chunks[:17]   # an odd final frame of 17 packets
    return b"".join(chunks), A


def _check_against_ref(h, r, dtype=np.float64, device=False):
    assert h.num_frames == len(r["frames"]) and h.num_packets == r["num_packets"] and h.bytes_used == r["bytes_used"]
    info = h.frame_info()
    for k, (n, t0, t1) in enumerate(r["info"]):
        assert info[k]["num_points"] == n
        assert (np.isnan(t0) and np.isnan(info[k]["t_first"])) or info[k]["t_first"] == t0
        assert (np.isnan(t1) and np.isnan(info[k]["t_max"])) or info[k]["t_max"] == t1
    got = h.read(dtype=dtype, device=device)
    xyz = np.concatenate([f[0] for f in r["frames"]])
    t = np.concatenate([f[1] for f in r["frames"]])
    if device:
        got = {k: v.cpu().numpy() for k, v in got.items()}
    assert np.array_equal(got["xyz"], xyz.astype(dtype)) and np.array_equal(got["t"], t)
    assert got["frame_ends"].tolist() == np.cumsum([f[1].size for f in r["frames"]]).tolist()
    return got


@pytest.mark.parametrize("device_sink", [False, True])
def test_nclt_decode_matches_the_restatement(eng, stream_bytes, device_sink):
    data, A = stream_bytes
    r = ref.decode(data, A, final=True)
    assert len(r["frames"]) == 4 and r["info"][-1][0] > 0
    h = eng.nclt_hits(data, A, final=True)
    _check_against_ref(h, r, device=device_sink)
    _check_against_ref(h, r, dtype=np.float32, device=device_sink)


def test_nclt_device_bytes_and_chunks_give_the_same_frames(eng, stream_bytes):
    import torch
    data, A = stream_bytes
    whole = eng.nclt_hits(data, A).read(device=False)
    dev = eng.nclt_hits(torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda(), A).read(device=False)
    for k in whole:
        assert np.array_equal(whole[k], dev[k]), k
    # whole-frame chunks of arbitrary byte sizes: bytes_used says where the next chunk starts
    for size in (30_000, 123_457, 400_001):
        pos, xyz, t = 0, [], []
        while pos < len(data):
            end = min(len(data), pos + size)
            final = end == len(data)
            h = eng.nclt_hits(data[pos:end], A, final=final)
            if h.num_frames:
                got = h.read(device=False)
                xyz.append(got["xyz"]), t.append(got["t"])
            if final:
                break
            if h.bytes_used == 0:
                size *= 2   # not one whole frame in this chunk: read more
                continue
            pos += h.bytes_used
        assert np.array_equal(np.concatenate(xyz), whole["xyz"]) and np.array_equal(np.concatenate(t), whole["t"])


def test_nclt_skipping_frames_equals_dropping_their_packets(eng, stream_bytes):
    data, A = stream_bytes
    packets, _, _ = ref.walk(data)
    h = eng.nclt_hits(data, A)
    for k in (1, 2):
        rest = data[packets[k * A][0]:]
        a = h.read(first=k, device=False)
        b = eng.nclt_hits(rest, A).read(device=False)
        for key in a:
            assert np.array_equal(a[key], b[key]), (k, key)


def test_nclt_magic_inside_a_hit_goes_through_the_walk(eng):
    """a hit (laser 173) whose 8 bytes equal the magic word: the chain check fails, the walk decodes it"""
    magic_hit = np.array([[44444, 44444, 44444]], dtype=np.uint16)
    pk = [ref.pack_packet(100, np.array([[1, 2, 3], [4, 5, 6]])),
          ref.pack_packet(101, np.concatenate([magic_hit, [[7, 8, 9]]]), laser=np.array([0xAD, 0]),
                          intensity=np.array([0x9C, 0])),
          ref.pack_packet(102, []), ref.pack_packet(103, np.array([[10, 11, 12]]))]
    data = b"".join(pk)
    assert data.count(b"\x9c\xad" * 4) == 4 + 1   # four headers and the hit
    r = ref.decode(data, 3, final=True)
    h = eng.nclt_hits(data, 3, final=True)
    _check_against_ref(h, r)
    assert h.read(device=False)["xyz"][2].tolist() == [44444 * 0.005 - 100.0] * 3


def test_nclt_refusals(eng, stream_bytes):
    data, A = stream_bytes
    packets, _, _ = ref.walk(data)
    bad = bytearray(data)
    off = packets[50][0]
    bad[off] ^= 1
    with pytest.raises(CticpError) as e:
        eng.nclt_hits(bytes(bad), A)
    assert e.value.code == abi.ERR_INVALID_ARGUMENT and ("byte offset %d " % off) in str(e.value)
    with pytest.raises(CticpError) as e:
        eng.nclt_hits(data[:-3], A, final=True)
    assert e.value.code == abi.ERR_INVALID_ARGUMENT and "truncated" in str(e.value)
    h = eng.nclt_hits(data[:-3], A, final=False)   # a partial last packet is left for the next chunk
    assert h.num_frames == 3 and h.bytes_used == packets[3 * A][0]
    with pytest.raises(CticpError):
        eng.nclt_hits(data, 0)
    with pytest.raises(CticpError):
        h.read(first=2, m=5, device=False)


def _ply_frames(rng, n, xdt, with_t, extra):
    fields = ([("intensity", "f4")] if extra else []) + [("x", xdt), ("y", xdt), ("z", xdt)] + \
        ([("timestamp", "f8")] if with_t else []) + ([("ring", "u2")] if extra else [])
    rec = np.zeros(n, dtype=fields)
    p = rng.uniform(-60, 60, (n, 3))
    p[:, 2] = rng.uniform(-8, 6, n)
    p[:7, :2] = 0.0                     # the z axis
    p[7:12, 2] = -5.0                   # exactly at the cut
    p[12, 2] = np.nan
    p[13, 0] = np.nan
    for k, c in enumerate("xyz"):
        rec[c] = p[:, k]
    if with_t:
        rec["timestamp"] = rng.uniform(0, 0.1, n)
    return rec


@pytest.mark.parametrize("xdt", ["f4", "f8"])
@pytest.mark.parametrize("with_t,extra", [(True, False), (False, True), (True, True)])
def test_kitti_filter_on_ply_frames_matches_the_restatement(eng, xdt, with_t, extra):
    import torch
    rng = np.random.default_rng(7)
    rec = _ply_frames(rng, 120_000, xdt, with_t, extra)
    lay, body = eng.ply_records(ref.ply_bytes(rec))
    xyz = np.stack([body["x"], body["y"], body["z"]], 1).astype(np.float64)
    want = ref.kitti_frame_filter(xyz).astype(xdt)
    host = eng.kitti_frame_filter(body)
    got = np.stack([host["x"], host["y"], host["z"]], 1)
    assert np.array_equal(got.view(np.uint8), want.view(np.uint8))
    keep = np.ones(lay.point_step, bool)   # every byte outside x, y, z kept
    keep[lay.xyz_offset:lay.xyz_offset + 3 * np.dtype(xdt).itemsize] = False
    assert np.array_equal(host.view(np.uint8).reshape(len(host), -1)[:, keep], body.view(np.uint8).reshape(len(body), -1)[:, keep])
    # in place on the device, on the records as they lie in the file
    raw = torch.from_numpy(body.view(np.uint8).reshape(len(body), -1).copy()).cuda()
    scan = abi.DeviceScan(raw.data_ptr() + lay.xyz_offset, lay.point_step, None, 0, len(body), lay.xyz_dtype, 0)
    sink = abi.CloudSink(raw.data_ptr(), len(body), lay.point_step, lay.xyz_offset, lay.xyz_dtype, 0, 0, 0)
    eng.check(eng.fn("kitti_frame_filter_device")(0, scan, sink, None))
    torch.cuda.synchronize()
    dev = raw.cpu().numpy().reshape(-1).view(body.dtype)
    assert np.array_equal(dev.view(np.uint8), host.view(np.uint8))
    tens = torch.from_numpy(xyz.astype(xdt)).cuda()
    assert np.array_equal(eng.kitti_frame_filter(tens).cpu().numpy(), want, equal_nan=True)   # the NaN point
    if with_t:
        ends = np.array([0, 40_000, 40_000, 119_999, 120_000], dtype=np.uint64)
        tt = body["t"]
        bounds = np.concatenate([[0], ends.astype(np.int64)])
        exp = np.array([[tt[a:b].min(), tt[a:b].max()] if b > a else [np.inf, -np.inf]
                        for a, b in zip(bounds[:-1], bounds[1:])])
        assert np.array_equal(eng.scan_time_ranges(tt, ends), exp)
        td = torch.from_numpy(np.ascontiguousarray(tt)).cuda()
        assert np.array_equal(eng.scan_time_ranges(td, torch.from_numpy(ends.astype(np.int64))).cpu().numpy(), exp)
        tt2 = tt.copy()
        tt2[50_000] = np.nan
        with pytest.raises(CticpError):
            eng.scan_time_ranges(tt2, ends)
        r = eng.scan_time_ranges(torch.from_numpy(tt2).cuda(), torch.from_numpy(ends.astype(np.int64))).cpu().numpy()
        assert np.isnan(r[3]).all() and np.array_equal(r[[0, 1, 2, 4]], exp[[0, 1, 2, 4]])


def test_decoded_nclt_frames_register_as_their_host_copy(eng):
    """frames decoded into device memory through register_device, against register_frame on the restatement's host
    decode of the same bytes: the same poses, bit for bit"""
    import torch
    m, A = 6, 220
    out, _ = _sweeps(eng, m, seed=5)
    data = b"".join(_pack(out, A, np.random.default_rng(2)))
    r = ref.decode(data, A)
    h = eng.nclt_hits(data, A)
    dev = h.read()
    ends = dev["frame_ends"].cpu().numpy()
    starts = np.concatenate([[0], ends[:-1]])
    rec = dev["xyz"].stride(0) * dev["xyz"].element_size()
    stream = torch.cuda.current_stream().cuda_stream
    od_d = eng.odometry(_sequence_options(eng, "GN", init_num_frames=3))
    od_h = eng.odometry(_sequence_options(eng, "GN", init_num_frames=3))
    for k in range(m):
        a, n = int(starts[k]), int(ends[k] - starts[k])
        scan = abi.DeviceScan(dev["xyz"].data_ptr() + a * rec, rec, dev["t"].data_ptr() + a * rec, rec, n,
                              abi.DTYPE["float64"], abi.DTYPE["float64"])
        sd = od_d.register_device(scan, k, stream=stream)
        sh = od_h.RegisterFrame(np.ascontiguousarray(r["frames"][k][0]), np.ascontiguousarray(r["frames"][k][1]), k)
        assert sd.success and sh.success, (k, sd.error_message, sh.error_message)
        for a_, b_ in ((sd.frame.begin_pose, sh.frame.begin_pose), (sd.frame.end_pose, sh.frame.end_pose)):
            assert list(a_.quat) == list(b_.quat) and list(a_.tr) == list(b_.tr), k
