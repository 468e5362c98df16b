"""Neighbourhoods on the device (cticp_neighborhood_*) against the CPU restatement of slam::TNeighborhood
(tests/oracle_neighborhood): the k-nearest search exactly (indices, d2 bits, counts), the descriptions within the error
model of the device eigen-solver, and the consistency of the host, device and world-cloud forms."""
import ctypes as C

import numpy as np
import pytest

import ct_icp_b200
import oracle_neighborhood_lib as orn
from ct_icp_b200 import _abi as abi

pytestmark = pytest.mark.gpu
DBL_MAX = np.finfo(np.float64).max
U = np.finfo(np.float64).eps / 2


def _lidar(n, seed=0, offset=(350.0, -120.0, 12.0)):
    rng = np.random.default_rng(seed)
    az = rng.uniform(0, 2 * np.pi, n)
    el = np.deg2rad(-25 + 28 * rng.integers(0, 64, n) / 63)
    wall = rng.uniform(5, 60, n)
    r_ground = np.where(el < -0.02, 1.7 / np.tan(-np.minimum(el, -1e-3)), 1e9)
    r = np.minimum(wall / np.cos(el), r_ground)
    return np.stack([r * np.cos(el) * np.cos(az), r * np.cos(el) * np.sin(az), r * np.sin(el)], 1) \
        + np.asarray(offset)


def _clouds():
    rng = np.random.default_rng(1)
    yield "random", rng.uniform(-5, 5, (20000, 3))
    yield "lidar", _lidar(30000)
    base = np.round(rng.uniform(-2, 2, (500, 3)), 1)
    yield "duplicates", base[rng.integers(0, 500, 5000)]


def _assert_search_equal(got, ref, what=""):
    gi, gd, gc = got
    ri, rd, rc = ref
    np.testing.assert_array_equal(gc, rc, err_msg=what)
    np.testing.assert_array_equal(gi, ri, err_msg=what)
    np.testing.assert_array_equal(gd.view(np.uint64), rd.view(np.uint64), err_msg=what)


@pytest.mark.parametrize("k", [1, 5, 10, 20, 32])
def test_search_matches_oracle(eng, k):
    for name, pts in _clouds():
        nb = eng.neighborhood(pts)
        rng = np.random.default_rng(k)
        c = pts.mean(0)
        q = np.concatenate([pts[rng.integers(0, len(pts), 300)] + rng.normal(0, 0.2, (300, 3)),
                            [c + [100.0, 0, 0], c + [0, 1e4, 0], c - [1e4, 1e4, 1e4]], [[np.nan, 0, 0], [0, 0, np.inf]]])
        _, d2u, _ = orn.search(pts, q[:50], k)
        cut = float(np.median(d2u[:, k // 2]))   # a radius that cuts many counts below k
        for r in (DBL_MAX, cut, 1e-6):
            _assert_search_equal(nb.search(q, k, r), orn.search(pts, q, k, r), f"{name} k={k} r={r}")
        sel = rng.integers(0, len(pts), 2000)   # self queries: the points themselves, in index order
        got = nb.search(None, k)
        ref = orn.search(pts, pts[sel], k)
        _assert_search_equal(tuple(a[sel] for a in got), ref, f"{name} self k={k}")


def test_search_ties_non_finite_and_small(eng):
    ring = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1], [0, 0, 0.]])
    for k in (1, 2, 3, 7, 10):
        _assert_search_equal(eng.neighborhood(ring).search(np.zeros((1, 3)), k), orn.search(ring, np.zeros((1, 3)), k))
    _assert_search_equal(eng.neighborhood(ring).search(np.zeros((1, 3)), 7, 1.0), orn.search(ring, np.zeros((1, 3)), 7, 1.0))
    rng = np.random.default_rng(2)
    pts = rng.uniform(0, 1, (3000, 3))
    bad = [3, 99, 2500]
    pts[bad] = [[np.nan, 0, 0], [np.inf, 1, 1], [0, -np.inf, 0]]
    nb = eng.neighborhood(pts)
    assert nb.num_points() == 3000 and nb.num_rejected() == 3
    got = nb.search(None, 12)
    _assert_search_equal(got, orn.search(pts, None, 12))
    assert (got[2][bad] == 0).all()
    for n in (0, 1, 4):
        p = rng.uniform(0, 1, (n, 3))
        q = rng.uniform(0, 1, (20, 3))
        _assert_search_equal(eng.neighborhood(p).search(q, 5), orn.search(p, q, 5))
    for r in (0.0, -1.0):
        assert (nb.search(pts[:10], 5, r)[2] == 0).all()


def test_search_20m_points_once(eng):
    rng = np.random.default_rng(9)
    pts = rng.uniform(-200, 200, (20_000_000, 3)) * [1, 1, 0.05]
    nb = eng.neighborhood(pts)
    q = np.array([[0.5, -3.0, 0.1], [1e4, 0, 0]])
    _assert_search_equal(nb.search(q, 32), orn.search(pts, q, 32))


def _desc_close(got, ref, what, centre):
    """the error model of test_gpu_device_math.py: eigenvalues within c u S, vectors within that over the gap, where S is
    lambda_1 plus the squared offset of the barycenter from the centre the device sums about (the query, or the set's
    first point): the rounding of the centred sums. Near-degenerate gaps and neighbourhoods with S >> lambda_1 (points
    that nearly coincide) skip the vectors and ratios."""
    assert got["is_valid"] == ref["is_valid"], what
    if not ref["is_valid"]:
        assert got.tobytes() == ref.tobytes(), what
        return
    cov = ref["covariance"]
    M = np.array([[cov[0], cov[1], cov[2]], [cov[1], cov[3], cov[4]], [cov[2], cov[4], cov[5]]])
    w = np.sort(np.abs(np.linalg.eigvalsh(M)))[::-1]
    S = w[0] + float(np.sum((ref["barycenter"] - np.asarray(centre)) ** 2))
    tol = 256 * U * max(S, 1e-300)
    np.testing.assert_allclose(got["covariance"], cov, rtol=0, atol=tol, err_msg=what)
    np.testing.assert_allclose(got["barycenter"], ref["barycenter"], rtol=1e-13, atol=1e-9, err_msg=what)
    if w[0] > 1e6 * tol:
        e = tol / w[0]   # relative error of the eigenvalues
        for field in ("linearity", "planarity"):
            assert abs(got[field] - ref[field]) <= 4 * e + 1e-12, (what, field, got[field], ref[field])
        assert abs(got["a2D"] - ref["a2D"]) <= 4 * np.sqrt(e) + 1e-9, what
        assert abs(got["cov_det"] - ref["cov_det"]) <= 8 * tol * w[0] ** 2 + 1e-300, what
        for field, gap in (("normal", w[1] - w[2]), ("line", w[0] - w[1])):
            if gap > 1e3 * tol:
                cosang = abs(np.dot(got[field], ref[field]))
                assert cosang >= 1 - 0.5 * (8 * tol / gap) ** 2 - 1e-15, (what, field, cosang)
        near = abs(ref["planarity"] - 0.8) < 8 * e or abs(ref["linearity"] - 0.8) < 8 * e
        if not near:
            assert got["type"] == ref["type"], what


@pytest.mark.parametrize("k", [5, 10, 20, 32])
def test_describe_matches_oracle(eng, k):
    for name, pts in _clouds():
        nb = eng.neighborhood(pts)
        rng = np.random.default_rng(k)
        q = np.concatenate([pts[rng.integers(0, len(pts), 150)] + rng.normal(0, 0.05, (150, 3)), pts[:50]])
        for r in (DBL_MAX, 0.3):
            got = nb.describe(q, k, r)
            idx, _, cnt = orn.search(pts, q, k, r)
            for i in range(len(q)):
                ref = orn.describe(pts[idx[i, :cnt[i]].astype(np.int64)], centre=q[i])
                _desc_close(got[i], ref, f"{name} k={k} r={r} q={i}", q[i])


def test_describe_near_origin_against_the_uncentred_formula(eng):
    pts = np.random.default_rng(4).normal(0, 1, (5000, 3)) * [2, 1, 0.3]
    nb = eng.neighborhood(pts)
    got = nb.describe(pts[:200], 20)
    idx, _, cnt = orn.search(pts, pts[:200], 20)
    for i in range(200):
        ref = orn.describe(pts[idx[i].astype(np.int64)], centred=False)
        np.testing.assert_allclose(got[i]["covariance"], ref["covariance"], rtol=0, atol=1e-13)
        assert abs(got[i]["planarity"] - ref["planarity"]) < 1e-10


def test_describe_values_subsets_nan_and_planar(eng):
    rng = np.random.default_rng(6)
    pts = rng.normal(0, 1, (2000, 3))
    nb = eng.neighborhood(pts)
    full = nb.describe(pts[:100], 20)
    for values in range(0, 128):
        d = nb.describe(pts[:100], 20, values=values)
        ref = np.array([orn.describe(pts[orn.search(pts, pts[i:i + 1], 20)[0][0].astype(np.int64)], values=values,
                                     centre=pts[i]) for i in range(3)])
        for f, bit in (("line", 1), ("normal", 2), ("planarity", 4), ("linearity", 8), ("cov_det", 16), ("a2D", 64)):
            if values & bit:
                np.testing.assert_array_equal(d[f], full[f])
            else:
                assert (d[f] == (-1 if f in ("planarity", "linearity", "cov_det", "a2D") else 0)).all(), (values, f)
        np.testing.assert_array_equal(d["type"][:3], ref["type"])
    same = np.tile([[10.0, 20.0, 30.0]], (8, 1))
    d = eng.neighborhood(same).describe(same[:1], 6)[0]
    assert d["is_valid"] == 1 and np.isnan(d["planarity"]) and np.isnan(d["linearity"]) and d["type"] == 0
    plane = rng.uniform(-1, 1, (10, 3))
    plane[:, 2] = 1.0
    s = eng.describe_point_sets(plane, values=abi.NB["ALL_BUT_KDTREE"])[0]
    assert abs(s["normal"][2]) == 1.0
    d = eng.neighborhood(plane).describe(plane[:1], 10, values=abi.NB["ALL_BUT_KDTREE"])[0]
    assert abs(d["normal"][2]) == 1.0


def test_describe_sets_matches_oracle(eng):
    rng = np.random.default_rng(8)
    pts = _lidar(20000, 3)
    ends = np.sort(rng.integers(0, len(pts), 300))
    ends = np.concatenate([[0, 3, 3, 8], ends, [len(pts)]]).astype(np.uint64)
    got = eng.describe_point_sets(pts, ends, values=abi.NB["ALL"])
    b = 0
    for s, e in enumerate(ends):
        _desc_close(got[s], orn.describe(pts[b:int(e)]), f"set {s}", pts[b] if int(e) > b else np.zeros(3))
        b = int(e)


def test_device_world_cloud_and_reruns_are_identical(eng):
    import torch
    pts = _lidar(200000, 5)
    nb = eng.neighborhood(pts)
    q = pts[::7] + 0.01
    host_s, host_d = nb.search(q, 20), nb.describe(q, 20)
    again = nb.search(q, 20), nb.describe(q, 20)
    for a, b in zip(host_s, again[0]):
        assert a.tobytes() == b.tobytes()
    assert host_d.tobytes() == again[1].tobytes()
    for dtype in (torch.float64, torch.float32):
        t = torch.tensor(pts, dtype=dtype, device="cuda")
        nbd = eng.neighborhood(t)
        ref_pts = t.double().cpu().numpy()
        nbh = eng.neighborhood(ref_pts)
        qd = torch.tensor(q, device="cuda")
        si, sd, sc = nbd.search(qd, 20)
        hi, hd, hc = nbh.search(q, 20)
        assert si.cpu().numpy().view(np.uint64).tobytes() == hi.tobytes()
        assert sd.cpu().numpy().tobytes() == hd.tobytes() and sc.cpu().numpy().tobytes() == hc.tobytes()
        dd = nbd.describe(qd, 20)
        torch.cuda.synchronize()
        assert dd.cpu().numpy().tobytes() == nbh.describe(q, 20).tobytes()
    wc = eng.world_cloud(0.1, 2)
    wc.add(pts[:100000])
    wc.add(pts[100000:])
    exported = wc.export()
    nw, ne = wc.neighborhood(), eng.neighborhood(exported)
    assert nw.num_points() == len(exported)
    assert nw.describe(None, 10).tobytes() == ne.describe(None, 10).tobytes()
    for a, b in zip(nw.search(None, 10), ne.search(None, 10)):
        assert a.tobytes() == b.tobytes()


def test_refusals_write_nothing(eng):
    import torch
    pts = np.random.default_rng(0).uniform(0, 1, (1000, 3))
    nb = eng.neighborhood(pts)
    q = pts[:10].copy()
    f = eng.fn("neighborhood_search")
    idx = np.full((10, 8), 7, dtype=np.uint64)
    d2 = np.full((10, 8), 7.0)
    cnt = np.full(10, 7, dtype=np.int32)

    def call(k=8, r=DBL_MAX, qp=q.ctypes.data, m=10, i=idx.ctypes.data, d=d2.ctypes.data, c=cnt.ctypes.data, h=None):
        return f(h if h is not None else nb.h, qp, m, k, r, i, d, c)

    for rc, code in ((call(k=0), abi.ERR_INVALID_ARGUMENT), (call(k=33), abi.ERR_UNSUPPORTED),
                     (call(r=float("nan")), abi.ERR_INVALID_ARGUMENT), (call(i=None), abi.ERR_INVALID_ARGUMENT),
                     (call(qp=None, m=10), abi.ERR_INVALID_ARGUMENT), (call(h=C.c_void_p()), abi.ERR_INVALID_ARGUMENT)):
        assert rc == code
    assert (idx == 7).all() and (d2 == 7.0).all() and (cnt == 7).all()
    out = torch.full((10, 8), 7, dtype=torch.int64, device="cuda")
    dd = torch.full((10, 8), 7.0, dtype=torch.float64, device="cuda")
    cc = torch.full((10,), 7, dtype=torch.int32, device="cuda")
    qd = torch.tensor(q, device="cuda")
    fd = eng.fn("neighborhood_search_device")
    def segment_end(ptr):   # the end of the caching allocator's segment that holds the tensor
        seg = next(g for g in torch.cuda.memory_snapshot() if g["address"] <= ptr < g["address"] + g["total_size"])
        return seg["address"] + seg["total_size"]

    near_end = segment_end(out.data_ptr()) - 10 * 8 * 8 + 8   # indices that would end 8 bytes past the allocation
    assert fd(nb.h, qd.data_ptr(), 10, 8, DBL_MAX, near_end, dd.data_ptr(), cc.data_ptr(), None) == \
        abi.ERR_INVALID_ARGUMENT
    assert fd(nb.h, q.ctypes.data, 10, 8, DBL_MAX, out.data_ptr(), dd.data_ptr(), cc.data_ptr(), None) == \
        abi.ERR_INVALID_ARGUMENT   # host memory as device queries
    torch.cuda.synchronize()
    assert (out == 7).all() and (dd == 7.0).all() and (cc == 7).all()
    fs = eng.fn("neighborhood_describe_sets")
    desc = np.zeros(2, dtype=abi.neighborhood_description_dtype())
    desc["planarity"] = 7.0
    bad_ends = np.array([600, 500], dtype=np.uint64)
    assert fs(0, pts.ctypes.data, 24, 1000, bad_ends.ctypes.data, 2, 127, 0.8, 0.8, desc.ctypes.data) == \
        abi.ERR_INVALID_ARGUMENT
    assert (desc["planarity"] == 7.0).all()


def test_describe_and_create_refusals_write_nothing(eng):
    import torch
    pts = np.random.default_rng(1).uniform(0, 1, (1000, 3))
    nb = eng.neighborhood(pts)
    q = pts[:10].copy()
    dt = abi.neighborhood_description_dtype()
    out = np.zeros(10, dtype=dt)
    out["planarity"] = 7.0
    f = eng.fn("neighborhood_describe")

    def call(k=8, r=DBL_MAX, o=out.ctypes.data, qp=q.ctypes.data, m=10):
        return f(nb.h, qp, m, k, r, 127, 0.8, 0.8, o)

    for rc, code in ((call(k=0), abi.ERR_INVALID_ARGUMENT), (call(k=33), abi.ERR_UNSUPPORTED),
                     (call(r=float("nan")), abi.ERR_INVALID_ARGUMENT), (call(o=None), abi.ERR_INVALID_ARGUMENT),
                     (call(qp=None, m=999), abi.ERR_INVALID_ARGUMENT)):
        assert rc == code
    assert (out["planarity"] == 7.0).all()
    fd = eng.fn("neighborhood_describe_device")
    qd = torch.tensor(q, device="cuda")
    od = torch.full((10 * dt.itemsize + 8,), 7, dtype=torch.uint8, device="cuda")

    def dcall(k=8, r=DBL_MAX, o=None, qp=None):
        return fd(nb.h, qp if qp is not None else qd.data_ptr(), 10, k, r, 127, 0.8, 0.8,
                  o if o is not None else od.data_ptr(), None)

    def segment_end(ptr):
        seg = next(g for g in torch.cuda.memory_snapshot() if g["address"] <= ptr < g["address"] + g["total_size"])
        return seg["address"] + seg["total_size"]

    for rc, code in ((dcall(k=0), abi.ERR_INVALID_ARGUMENT), (dcall(k=33), abi.ERR_UNSUPPORTED),
                     (dcall(r=float("nan")), abi.ERR_INVALID_ARGUMENT),
                     (dcall(o=od.data_ptr() + 4), abi.ERR_INVALID_ARGUMENT),                  # misaligned records
                     (dcall(qp=qd.data_ptr() + 4), abi.ERR_INVALID_ARGUMENT),                 # misaligned queries
                     (dcall(o=segment_end(od.data_ptr()) - 10 * dt.itemsize + 8), abi.ERR_INVALID_ARGUMENT),
                     (dcall(o=out.ctypes.data), abi.ERR_INVALID_ARGUMENT),                   # host memory
                     (dcall(qp=q.ctypes.data), abi.ERR_INVALID_ARGUMENT)):
        assert rc == code
    torch.cuda.synchronize()
    assert (od == 7).all()
    fs = eng.fn("neighborhood_search_device")
    idx = torch.full((10 * 8 + 1,), 7, dtype=torch.int64, device="cuda")
    dd = torch.full((10 * 8,), 7.0, dtype=torch.float64, device="cuda")
    cc = torch.full((10,), 7, dtype=torch.int32, device="cuda")
    assert fs(nb.h, qd.data_ptr(), 10, 8, DBL_MAX, idx.data_ptr() + 4, dd.data_ptr(), cc.data_ptr(), None) == \
        abi.ERR_INVALID_ARGUMENT   # misaligned indices
    torch.cuda.synchronize()
    assert (idx == 7).all() and (dd == 7.0).all() and (cc == 7).all()
    # create_device: an unknown dtype, host memory, a scan past its allocation
    fc = eng.fn("neighborhood_create_device")
    t = torch.tensor(pts, device="cuda")
    h = C.c_void_p()
    for scan in (abi.DeviceScan(t.data_ptr(), 24, None, 0, 1000, 6, 0),
                 abi.DeviceScan(pts.ctypes.data, 24, None, 0, 1000, abi.DTYPE["float64"], 0),
                 abi.DeviceScan(segment_end(t.data_ptr()) - 1000 * 24 + 8, 24, None, 0, 1000, abi.DTYPE["float64"], 0)):
        assert fc(C.byref(scan), None, 0, C.byref(h)) == abi.ERR_INVALID_ARGUMENT
        assert not h.value
