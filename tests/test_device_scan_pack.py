"""The packing format of a scan (csrc/scan_pack.cuh), shared by the host loops and the kernels of a scan in device memory,
built with plain g++ and compared with a NumPy restatement: hi / lo planes, alpha, needs-lo, timestamp min / max and the
rebuilt timestamps, for both x, y, z dtypes, every timestamp dtype and unaligned record layouts."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = {1: np.int8, 2: np.uint8, 3: np.int16, 4: np.uint16, 5: np.int32, 6: np.uint32, 7: np.float32, 8: np.float64}


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    out = str(tmp_path_factory.mktemp("scan_pack") / "scan_pack_test")
    r = subprocess.run([cxx, "-std=c++17", "-O2", "-Wall", "-Werror", "-I", os.path.join(ROOT, "ct_icp_b200", "csrc"),
                        os.path.join(ROOT, "tests", "cpp", "scan_pack_test.cpp"), "-o", out], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out


def _records(n, step, xoff, xdt, toff, tdt, xyz, t):
    buf = np.zeros(n * step, dtype=np.uint8)
    x = np.ndarray((n, 3), dtype=DTYPES[xdt], buffer=buf, offset=xoff, strides=(step, np.dtype(DTYPES[xdt]).itemsize))
    x[:] = xyz
    tt = np.ndarray((n,), dtype=DTYPES[tdt], buffer=buf, offset=toff, strides=(step,))
    tt[:] = t
    return buf


def _restated(xyz, t, xdt, pose):
    """What the engine packs, restated with NumPy's IEEE float64 (no fused multiply-add)."""
    t = t.astype(np.float64)
    valid = t[~np.isnan(t)]
    mn_s, mx_s = (valid.min(), valid.max()) if len(valid) else (np.inf, -np.inf)
    b, e = pose if pose is not None else (mn_s, mx_s)
    mn, mx = min(b, e), max(b, e)
    spans = mx > mn
    inv = 1.0 / (mx - mn) if spans else 0.0
    with np.errstate(invalid="ignore"):
        a = (t - mn) * inv if spans else np.ones_like(t)
    v = np.concatenate([xyz.astype(np.float64), a[:, None]], axis=1)
    hi = v.astype(np.float32)
    lo = (v - hi.astype(np.float64)).astype(np.float32)
    needs_lo = xdt == 8 and bool(np.any(hi[:, :3].astype(np.float64) != v[:, :3]))
    back = hi.astype(np.float64) + (lo.astype(np.float64) if needs_lo else 0.0)
    with np.errstate(invalid="ignore"):
        ts = mn + (hi[:, 3].astype(np.float64) + (lo[:, 3].astype(np.float64) if needs_lo else 0.0)) * (mx - mn)
    back[:, 3] = ts
    return mn_s, mx_s, needs_lo, hi, lo, back


def _run(exe, tmp_path, n, step, xoff, xdt, toff, tdt, xyz, t, pose=None):
    buf = _records(n, step, xoff, xdt, toff, tdt, xyz, t)
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    buf.tofile(fin)
    b, e = pose if pose is not None else (0.0, 0.0)
    r = subprocess.run([exe, fin, fout, str(n), str(step), str(xoff), str(xdt), str(toff), str(tdt),
                        "1" if pose is not None else "0", float(b).hex(), float(e).hex()], capture_output=True, text=True)
    assert r.returncode == 0 and "SCAN PACK OK" in r.stdout, r.stdout + r.stderr
    raw = np.fromfile(fout, dtype=np.uint8)
    mn, mx = np.frombuffer(raw[:16].tobytes(), dtype=np.float64)
    needs_lo = int(np.frombuffer(raw[16:20].tobytes(), dtype=np.int32)[0])
    rec = np.frombuffer(raw[24:].tobytes(), dtype=[("hi", "<f4", 4), ("lo", "<f4", 4), ("back", "<f8", 4)])
    assert len(rec) == n
    # the stored values, in the scalar type the engine reads
    xs = np.ndarray((n, 3), dtype=DTYPES[xdt], buffer=buf, offset=xoff, strides=(step, np.dtype(DTYPES[xdt]).itemsize))
    ts = np.ndarray((n,), dtype=DTYPES[tdt], buffer=buf, offset=toff, strides=(step,))
    want = _restated(np.array(xs), np.array(ts), xdt, pose)
    assert mn == want[0] and mx == want[1]
    assert bool(needs_lo) == want[2]
    assert rec["hi"].tobytes() == want[3].tobytes()
    if want[2]:
        assert rec["lo"].tobytes() == want[4].tobytes()
    assert rec["back"].tobytes() == want[5].tobytes()
    return want


def _scan(rng, n, t0=1000.0, span=0.1):
    xyz = rng.uniform(-80.0, 80.0, size=(n, 3))
    t = t0 + np.sort(rng.uniform(0.0, span, size=n))
    return xyz, t


@pytest.mark.parametrize("tdt", sorted(DTYPES))
@pytest.mark.parametrize("xdt", [7, 8])
def test_every_dtype_packed_layout(exe, tmp_path, xdt, tdt):
    rng = np.random.default_rng(100 * xdt + tdt)
    n = 257
    xyz, _ = _scan(rng, n)
    if DTYPES[tdt] in (np.float32, np.float64):
        t = 50.0 + np.sort(rng.uniform(0.0, 0.1, size=n))
    else:   # integer timestamps (e.g. nanosecond offsets) within the type's range
        info = np.iinfo(DTYPES[tdt])
        t = np.sort(rng.integers(max(info.min, -100), min(info.max, 120), size=n))
    xsz = np.dtype(DTYPES[xdt]).itemsize
    tsz = np.dtype(DTYPES[tdt]).itemsize
    # point_step 21-ish: x at byte 1, t right behind z, nothing aligned
    step = 1 + 3 * xsz + tsz + 2
    _run(exe, tmp_path, n, step, 1, xdt, 1 + 3 * xsz, tdt, xyz, t)


@pytest.mark.parametrize("xdt", [7, 8])
def test_point_step_21_x_at_byte_1(exe, tmp_path, xdt):
    rng = np.random.default_rng(21)
    xyz, t = _scan(rng, 300)
    if xdt == 8:   # 1 + 24 > 21: a float64 record needs more room
        _run(exe, tmp_path, 300, 37, 1, 8, 29, 8, xyz, t)
    else:
        _run(exe, tmp_path, 300, 21, 1, 7, 13, 8, xyz, t)


def test_constant_timestamps_give_alpha_one(exe, tmp_path):
    rng = np.random.default_rng(3)
    xyz, _ = _scan(rng, 64)
    want = _run(exe, tmp_path, 64, 32, 0, 8, 24, 8, xyz, np.full(64, 7.25))
    assert np.all(want[3][:, 3] == 1.0)


def test_float64_values_float32_cannot_hold(exe, tmp_path):
    rng = np.random.default_rng(4)
    xyz, t = _scan(rng, 500)
    xyz[::7] += 1e-9                # not float32-representable: the residual plane is needed
    want = _run(exe, tmp_path, 500, 33, 1, 8, 25, 8, xyz, t)
    assert want[2]
    # a float64 scan of float32 values needs none
    want = _run(exe, tmp_path, 500, 32, 0, 8, 24, 8, xyz.astype(np.float32).astype(np.float64), t)
    assert not want[2]


def test_estimate_timestamps_and_nan_timestamps(exe, tmp_path):
    rng = np.random.default_rng(5)
    xyz, t = _scan(rng, 200)
    t[17] = np.nan                  # skipped by min / max, as by the host's comparisons
    _run(exe, tmp_path, 200, 32, 0, 8, 24, 8, xyz, t)
    _run(exe, tmp_path, 200, 32, 0, 8, 24, 8, xyz, t, pose=(t[1] + 0.05, t[0] - 0.01))   # reversed pair


def test_device_scan_struct_size():
    import ct_icp_b200
    from ct_icp_b200 import _abi as abi
    eng = ct_icp_b200.engine()
    assert eng.fn("abi_sizeof")(b"cticp_device_scan") == C.sizeof(abi.DeviceScan) == 48
