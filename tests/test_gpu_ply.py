"""PLY files on the device (include/cticp.h, "PLY files") against the CPU oracle (tests/oracle_ply, a restatement of
WriteCollectionToPLY over tinyply 2.x): bytes equal bit for bit for every source x PLY type, record sizes, strides,
alignments and output phases; many files per call with their offsets, capacities and clamped ends; a call past 4 GiB;
stream order; round trips through the readers; and the refusals."""
import ctypes as C
import os
import sys
import tempfile

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import oracle_ply_lib as orc  # noqa: E402
import ply_ref  # noqa: E402

from ct_icp_b200 import _abi as abi  # noqa: E402
from ct_icp_b200 import datasets  # noqa: E402
from ct_icp_b200 import synthetic as syn  # noqa: E402
from ct_icp_b200._binding import CticpError  # noqa: E402
import lidar_sim_ref as lref  # noqa: E402

pytestmark = pytest.mark.gpu

SRC = ["int8", "uint8", "int16", "uint16", "int32", "uint32", "float32", "float64", "int64", "uint64"]


def _cuda(a):
    import torch
    return torch.from_numpy(np.array(a)).cuda()   # np.array keeps a 0-d value 0-d


def _values(rng, dtype, n):
    dt = np.dtype(dtype)
    if dt.kind == "f":
        v = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 12, n)
        v[rng.random(n) < 0.05] = np.nan
        v[::7] = np.round(v[::7]) + 0.5
        v[::11] = -v[::11]
        return v.astype(dt)
    info = np.iinfo(dt)
    return rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)


def _raw(eng, props, n, ends, m, out, cap, offsets, stream=None):
    """cticp_ply_write_device with raw (element, name, ply, src, ptr, stride) tuples"""
    arr = (abi.PlyProperty * max(len(props), 1))()
    keep = []
    for i, (e, nm, ply, src, ptr, stride) in enumerate(props):
        keep += [e.encode(), nm.encode()]
        arr[i] = abi.PlyProperty(keep[-2], keep[-1], ply, src, ptr, stride)
    return eng.fn("ply_write_device")(0, arr if props else None, len(props), n, ends, m, out, cap, offsets,
                                      C.c_void_p(stream))


@pytest.mark.parametrize("src", SRC)
def test_every_dtype_pair_equals_the_oracle(eng, src):
    rng = np.random.default_rng(abi.PLY_SRC_DTYPE[src] + 40)
    for n in (0, 1, 1000):
        vals = _values(rng, src, n)
        cols = [("vertex", "p%d" % ply, ply, vals) for ply in range(1, 9)]
        want = orc.ply_write(cols)
        out, off = eng.ply_write([c[:3] + (_cuda(c[3]),) for c in cols])
        assert out.cpu().numpy().tobytes() == want and off.tolist() == [0, len(want)], (src, n)
        assert eng.ply_write(cols) == want                     # the host variant, through the same kernels


def test_fp64_ties_negative_to_unsigned_and_saturation(eng):
    ties = np.array([1.0 + 2.0 ** -24, 1.0 + 3 * 2.0 ** -24, -(1.0 + 2.0 ** -24), 2.0 ** 127 * (2 - 2.0 ** -24)])
    out, _ = eng.ply_write([("v", "x", "float", _cuda(ties))])
    assert out.cpu().numpy().tobytes() == orc.ply_write([("v", "x", "float", ties)])
    neg = np.array([-1, -128, -129, -2 ** 31], dtype=np.int64)
    cols = [("v", "a", "uchar", neg), ("v", "b", "ushort", neg), ("v", "c", "uint", neg)]
    body = eng.ply_write(cols)[-4 * 7:]
    rec = np.frombuffer(body, dtype=[("a", "u1"), ("b", "<u2"), ("c", "<u4")])
    assert rec["a"].tolist() == [255, 128, 127, 0] and rec["c"].tolist() == [2 ** 32 - 1, 2 ** 32 - 128,
                                                                             2 ** 32 - 129, 2 ** 31]
    x = np.array([np.nan, 1e30, -1e30, 255.9, -0.9, -1.5, 3e9, np.inf, -np.inf])
    out, _ = eng.ply_write([("v", "u8", "uchar", _cuda(x)), ("v", "i32", "int", _cuda(x)),
                            ("v", "u32", "uint", _cuda(x.astype(np.float32)))])
    rec = np.frombuffer(out.cpu().numpy().tobytes()[-len(x) * 9:], dtype=[("u8", "u1"), ("i32", "<i4"), ("u32", "<u4")])
    assert rec["u8"].tolist() == [0, 255, 0, 255, 0, 0, 255, 255, 0]
    assert rec["i32"].tolist() == [0, 2 ** 31 - 1, -2 ** 31, 255, 0, -1, 2 ** 31 - 1, 2 ** 31 - 1, -2 ** 31]
    assert rec["u32"].tolist() == [0, 2 ** 32 - 1, 0, 255, 0, 0, 3000000000, 2 ** 32 - 1, 0]


@pytest.mark.parametrize("layout", ["1", "13", "20", "80", "256", "elements"])
def test_record_sizes_and_elements(eng, layout):
    rng = np.random.default_rng(len(layout))
    n = 5001
    f64 = lambda: rng.standard_normal(n)  # noqa: E731
    cols = {
        "1": [("vertex", "c", "uchar", rng.integers(0, 256, n, dtype=np.uint8))],
        "13": [("vertex", k, "float", f64()) for k in "xyz"] + [("vertex", "i", "uchar", rng.integers(0, 9, n))],
        "20": [("vertex", k, "float", f64()) for k in "xyz"] + [("vertex", "t", "double", f64())],
        "80": None,
        "256": [("vertex", "d%d" % i, "double", f64()) for i in range(32)],
        "elements": [("a", "x", "short", rng.integers(-9, 9, n)), ("b", "y", "double", f64()),
                     ("a", "z", "float", f64()), ("c", "w", "uchar", np.asarray(np.uint8(3)))],
    }[layout]
    if cols is None:
        poses = np.zeros(n, dtype=abi.pose_dtype())
        poses.view(np.uint8)[:] = rng.integers(0, 256, poses.nbytes, dtype=np.uint8)
        want = orc.save_poses_ply(poses)
        assert eng.save_poses_ply(poses) == want
        return
    want = orc.ply_write(cols, num_items=n)
    out, _ = eng.ply_write([c[:3] + (_cuda(c[3]),) for c in cols], num_items=n)
    assert out.cpu().numpy().tobytes() == want


def test_stride_zero_unaligned_sources_and_every_output_phase(eng):
    import torch
    rng = np.random.default_rng(9)
    n = 3001
    host = rng.integers(0, 256, 16 * n + 64, dtype=np.uint8)
    dev = _cuda(host)
    base = dev.data_ptr()
    # (element, name, ply, src dtype, byte offset, stride)
    spec = [("vertex", "x", 7, 8, 1, 13), ("vertex", "y", 8, 7, 3, 13), ("vertex", "i", 5, 3, 7, 15),
            ("vertex", "k", 2, 10, 5, 0), ("extra", "u", 6, 9, 2, 16)]
    ocols = []
    for e, nm, ply, sdt, off, stride in spec:
        name = [k for k, v in abi.PLY_SRC_DTYPE.items() if v == sdt][0]
        size = np.dtype(name).itemsize
        vals = np.array([host[off + i * stride: off + i * stride + size].view(name)[0] for i in range(n)])
        ocols.append((e, nm, ply, vals))
    want = orc.ply_write(ocols)
    ends = torch.tensor([n], dtype=torch.int64, device="cuda")
    offs = torch.empty(2, dtype=torch.int64, device="cuda")
    buf = torch.full((len(want) + 64,), 0xAB, dtype=torch.uint8, device="cuda")
    props = [(e, nm, ply, sdt, base + off, stride) for e, nm, ply, sdt, off, stride in spec]
    for phase in range(16):
        buf.fill_(0xAB)
        assert _raw(eng, props, n, ends.data_ptr(), 1, buf.data_ptr() + phase, len(want), offs.data_ptr()) == 0
        got = buf.cpu().numpy()
        assert got[phase:phase + len(want)].tobytes() == want, phase
        assert (got[:phase] == 0xAB).all() and (got[phase + len(want):] == 0xAB).all(), phase


def test_a_thousand_files_offsets_capacities(eng):
    import torch
    rng = np.random.default_rng(11)
    counts = rng.integers(0, 300, 1000)
    counts[rng.random(1000) < 0.1] = 0
    ends = np.cumsum(counts)
    n = int(ends[-1])
    xyz, t, idx = rng.standard_normal((n, 3)), rng.random(n), rng.integers(0, 2 ** 40, n, dtype=np.uint64)
    cols = [("vertex", k, "float", xyz[:, i]) for i, k in enumerate("xyz")] + [("vertex", "t", "double", t)] + \
        [("index", "i", "uint", idx)]
    files = [orc.ply_write([c[:3] + (c[3][b:e],) for c in cols], num_items=e - b)
             for b, e in zip(np.concatenate([[0], ends[:-1]]), ends)]
    want_off = np.concatenate([[0], np.cumsum([len(f) for f in files])])
    dcols = [c[:3] + (_cuda(c[3]),) for c in cols]
    out, off = eng.ply_write(dcols, file_ends=ends)
    assert off.cpu().numpy().tolist() == want_off.tolist()
    data = out.cpu().numpy().tobytes()
    for k in range(1000):
        assert data[want_off[k]:want_off[k + 1]] == files[k], k
    # capacity 0: the offsets only; a partial capacity: exactly the prefix
    props = [(e, nm, {"float": 7, "double": 8, "uint": 6}[p], abi.PLY_SRC_DTYPE[str(a.dtype).replace("torch.", "")],
              a.data_ptr(), a.stride(0) * a.element_size()) for e, nm, p, a in dcols]
    ends_d = torch.from_numpy(ends.astype(np.int64)).cuda()
    offs = torch.full((1001,), -1, dtype=torch.int64, device="cuda")
    buf = torch.full((len(data),), 0xAB, dtype=torch.uint8, device="cuda")
    assert _raw(eng, props, n, ends_d.data_ptr(), 1000, buf.data_ptr(), 0, offs.data_ptr()) == 0
    assert offs.cpu().numpy().tolist() == want_off.tolist() and bool((buf == 0xAB).all())
    for cap in (1, len(data) // 2 + 7, len(data) - 1):
        buf.fill_(0xAB)
        assert _raw(eng, props, n, ends_d.data_ptr(), 1000, buf.data_ptr(), cap, offs.data_ptr()) == 0
        got = buf.cpu().numpy()
        assert got[:cap].tobytes() == data[:cap] and (got[cap:] == 0xAB).all(), cap


def test_bad_file_ends_are_clamped_on_the_device_and_refused_on_the_host(eng):
    rng = np.random.default_rng(12)
    n = 10
    x = rng.standard_normal(n)
    ends = [5, 3, 100000, 8, 2 ** 62]
    clamped = [5, 5, 10, 10, 10]
    out, off = eng.ply_write([("vertex", "x", "double", _cuda(x))], file_ends=ends)
    files = [orc.ply_write([("vertex", "x", "double", x[b:e])], num_items=e - b)
             for b, e in zip([0] + clamped[:-1], clamped)]
    assert out.cpu().numpy().tobytes() == b"".join(files)
    assert off.cpu().numpy().tolist() == np.concatenate([[0], np.cumsum([len(f) for f in files])]).tolist()
    for bad in ([5, 3], [11]):
        with pytest.raises(CticpError) as e:
            eng.ply_write([("vertex", "x", "double", x)], file_ends=bad)
        assert e.value.code == abi.ERR_INVALID_ARGUMENT


def test_a_call_past_four_gib(eng):
    import torch
    # 5-byte records (float + uchar) of stride-0 columns; three files, the total past 2^32
    ends = [100_000_000, 550_000_000, 900_000_001]
    x, c = np.float32(1.5), np.uint8(7)
    cols = [("vertex", "x", "float", torch.tensor(1.5, dtype=torch.float32, device="cuda")),
            ("vertex", "c", "uchar", torch.tensor(7, dtype=torch.uint8, device="cuda"))]
    out, off = eng.ply_write(cols, file_ends=ends, num_items=ends[-1])
    counts = np.diff([0] + ends)
    heads = [ply_ref.header([("vertex", int(k), [("x", 7), ("c", 2)])]) for k in counts]
    want_off = np.concatenate([[0], np.cumsum([len(h) + 5 * k for h, k in zip(heads, counts)])])
    assert off.cpu().numpy().tolist() == want_off.tolist() and want_off[-1] > 2 ** 32
    rec = np.frombuffer(x.tobytes() + c.tobytes(), dtype=np.uint8)

    def expect(lo, hi):
        b = bytearray()
        for pos in range(lo, hi):
            k = int(np.searchsorted(want_off, pos, side="right") - 1)
            r = pos - want_off[k]
            b.append(heads[k][r] if r < len(heads[k]) else int(rec[(r - len(heads[k])) % 5]))
        return bytes(b)

    for lo in [0, int(want_off[1]) - 40, int(want_off[2]) - 3, 2 ** 32 - 4099, 2 ** 32 + 13, int(want_off[3]) - 300]:
        hi = min(lo + 4200, int(want_off[3]))
        assert out[lo:hi].cpu().numpy().tobytes() == expect(lo, hi), lo
    del out


def test_sources_written_on_a_side_stream(eng):
    import torch
    s = torch.cuda.Stream()
    n = 1 << 22
    with torch.cuda.stream(s):
        src = torch.arange(n, device="cuda", dtype=torch.float64).mul_(0.37).sin_()
        torch.cuda._sleep(20_000_000)
        src.add_(1.0)
        out, off = eng.ply_write([("vertex", "v", "float", src), ("vertex", "w", "int", src * 1000)])
        got = out.cpu().numpy().tobytes()
    h = src.cpu().numpy()
    assert got == orc.ply_write([("vertex", "v", "float", h), ("vertex", "w", "int", h * 1000)])


def test_sweeps_to_a_ply_directory_and_back(eng):
    import torch
    scene, traj = syn.UrbanScene(1234, profile="suburb"), syn.Trajectory(height=1.0)
    sc = eng.lidar_scene(scene.boxes, scene.cyl)
    m = 6
    tr = eng.continuous_trajectory(lref.trajectory_poses(traj, m * 0.1 + 0.2))
    out = sc.sweeps(tr, syn.HDL32, [(k * syn.HDL32.period, k) for k in range(m)], seed=4)
    ends = out["frame_ends"]
    with tempfile.TemporaryDirectory() as d:
        paths = datasets.write_ply_frames(eng, out["xyz"], out["t"], ends, d)
        assert [os.path.basename(p) for p in paths] == ["frame_%04d.ply" % k for k in range(m)]
        seq = datasets.PLYDirectory(eng, d, m)
        e = np.concatenate([[0], ends.cpu().numpy()]).astype(np.int64)
        xyz, t = out["xyz"].cpu().numpy(), out["t"].cpu().numpy()
        for k in range(m):
            with open(paths[k], "rb") as f:
                lay = eng.ply_layout(f.read())
            assert lay.num_points == e[k + 1] - e[k] and lay.xyz_dtype == abi.DTYPE["float32"]
            fr = seq._read(k)
            assert np.array_equal(fr["xyz"].cpu().numpy(), xyz[e[k]:e[k + 1]].astype(np.float32))
            assert np.array_equal(fr["t"].cpu().numpy(), t[e[k]:e[k + 1]].astype(np.float32).astype(np.float64))


def test_world_cloud_export_ply(eng):
    rng = np.random.default_rng(13)
    xyz = rng.uniform(-20, 20, (20000, 3))
    t = rng.random(20000)
    wc = eng.world_cloud(0.5, 2)
    wc.add(xyz, t)
    for dtype in (np.float32, np.float64):
        data = wc.export_ply(dtype, with_timestamps=True)
        _, rec = eng.ply_records(data)
        ref = wc.export(dtype, with_timestamps=True)
        assert np.array_equal(np.stack([rec["x"], rec["y"], rec["z"], rec["t"]], 1), ref)
    pts, src = wc.export(np.float64, with_timestamps=True, with_source_index=True)
    desc = wc.neighborhood().describe(k=8)
    data = wc.export_ply(np.float32, with_timestamps=True, with_source_index=True, normals=desc)
    cols = [("vertex", k, "float", pts[:, i]) for i, k in enumerate("xyz")] + \
        [("vertex", "timestamp", "float", pts[:, 3]), ("vertex", "source_index", "uint", src)] + \
        [("vertex", k, "float", desc["normal"][:, i]) for i, k in enumerate(("nx", "ny", "nz"))]
    assert data == orc.ply_write(cols)


def test_poses_round_trip(eng):
    rng = np.random.default_rng(14)
    poses = np.zeros(257, dtype=abi.pose_dtype())
    poses["quat"], poses["tr"] = rng.standard_normal((257, 4)), rng.standard_normal((257, 3))
    poses["ref_timestamp"], poses["dest_timestamp"] = rng.random(257), rng.random(257)
    poses["ref_frame_id"] = rng.integers(0, 2 ** 32, 257, dtype=np.uint32)
    poses["dest_frame_id"] = 0xFFFFFFFF
    data = eng.save_poses_ply(poses)
    assert data == orc.save_poses_ply(poses)
    assert eng.read_poses_ply(data).tobytes() == poses.tobytes()
    assert eng.save_poses_ply(poses[:0]) == orc.save_poses_ply(poses[:0])


def _segment_end(ptr):   # the caching allocator's segment that holds the tensor: the allocation the check sees
    import torch
    seg = next(g for g in torch.cuda.memory_snapshot() if g["address"] <= ptr < g["address"] + g["total_size"])
    return seg["address"] + seg["total_size"]


def test_refusals_enqueue_nothing(eng):
    import torch
    n = 100
    x = torch.zeros(n, dtype=torch.float64, device="cuda")
    short = _segment_end(x.data_ptr()) - 8 * n + 8          # n doubles that end 8 bytes past the segment
    host = np.zeros(n)
    ends = torch.tensor([n], dtype=torch.int64, device="cuda")
    offs = torch.full((2,), -1, dtype=torch.int64, device="cuda")
    buf = torch.full((4096,), 0xAB, dtype=torch.uint8, device="cuda")
    good = ("vertex", "x", 8, 8, x.data_ptr(), 8)
    E, B, O = ends.data_ptr(), buf.data_ptr(), offs.data_ptr()
    assert _raw(eng, [good], n, E, 1, B, 4096, O) == 0      # the good call works
    buf.fill_(0xAB)
    offs.fill_(-1)
    cases = [
        ([], n, E, 1, B, 4096, O),                                           # n_props 0
        ([good] + [("vertex", "p%d" % i, 8, 8, x.data_ptr(), 8) for i in range(32)], n, E, 1, B, 4096, O),
        ([("vertex", "x", 0, 8, x.data_ptr(), 8)], n, E, 1, B, 4096, O),     # unknown ply dtype
        ([("vertex", "x", 9, 8, x.data_ptr(), 8)], n, E, 1, B, 4096, O),     # INT64 is not a PLY type
        ([("vertex", "x", 8, 11, x.data_ptr(), 8)], n, E, 1, B, 4096, O),    # unknown source dtype
        ([("vertex", "", 8, 8, x.data_ptr(), 8)], n, E, 1, B, 4096, O),      # empty name
        ([("", "x", 8, 8, x.data_ptr(), 8)], n, E, 1, B, 4096, O),
        ([("vertex", "a" * 64, 8, 8, x.data_ptr(), 8)], n, E, 1, B, 4096, O),  # 64 bytes
        ([("vertex", "a b", 8, 8, x.data_ptr(), 8)], n, E, 1, B, 4096, O),   # whitespace
        ([("ver\ttex", "x", 8, 8, x.data_ptr(), 8)], n, E, 1, B, 4096, O),
        ([good, good], n, E, 1, B, 4096, O),                                 # the same property twice
        ([("vertex", "x", 8, 8, None, 8)], n, E, 1, B, 4096, O),             # null source
        ([("vertex", "x", 8, 8, host.ctypes.data, 8)], n, E, 1, B, 4096, O),  # host memory
        ([("vertex", "x", 8, 8, short, 8)], n, E, 1, B, 4096, O),            # past its allocation
        ([good], n, None, 1, B, 4096, O),                                    # null file_ends
        ([good], n, _segment_end(E) - 8, 2, B, 4096, O),                      # file_ends past its allocation
        ([good], n, E + 1, 1, B, 4096, O),                                   # unaligned
        ([good], n, E, 1, _segment_end(B) - 4095, 4096, O),                   # out past its allocation
        ([good], n, E, 1, None, 4096, O),                                    # null out with a capacity
        ([good], n, E, 1, B, 4096, None),                                    # null file_offsets
        ([good], n, E, 1, B, 4096, _segment_end(O) - 8),                      # file_offsets past its allocation
    ]
    for i, case in enumerate(cases):
        assert _raw(eng, *case) == abi.ERR_INVALID_ARGUMENT, i
    assert eng.fn("ply_write_device")(0, None, 1, n, E, 1, B, 4096, O, None) == abi.ERR_INVALID_ARGUMENT
    torch.cuda.synchronize()
    assert bool((buf == 0xAB).all()) and offs.tolist() == [-1, -1]


def test_existing_entry_points_refuse_64_bit_integer_types(eng):
    """CTICP_DTYPE_INT64 / UINT64 belong to cticp_ply_property only"""
    rec = np.zeros(4, dtype=[("x", "<f8"), ("y", "<f8"), ("z", "<f8"), ("t", "<i8")])
    ends = np.array([4], dtype=np.uint64)
    out = np.zeros((1, 2))
    for code in (9, 10):
        view = abi.CloudView(rec.ctypes.data, 4, 32, 0, abi.DTYPE["float64"], 24, code, 0)
        assert eng.fn("scan_time_ranges")(0, C.byref(view), ends.ctypes.data, 1, out.ctypes.data) == \
            abi.ERR_INVALID_ARGUMENT
