"""The CPU restatement of slam::TNeighborhood (tests/oracle_neighborhood) against independent NumPy statements: the
k-nearest search with a bound on d2 (np.lexsort on (index, d2)), every branch of ClassifyNeighborhood, the reference's
unit cases; the ctypes layout of cticp_neighborhood_description; and the engine's entry points failing loudly without a
GPU (CTICP_ERR_NO_DEVICE)."""
import ctypes as C

import numpy as np
import pytest

import ct_icp_b200
import oracle_neighborhood_lib as orn
from ct_icp_b200 import _abi as abi

DBL_MAX = np.finfo(np.float64).max


def numpy_knn(points, queries, k, max_radius=DBL_MAX):
    """independent statement: d2 = ((dx dx + dy dy) + dz dz), kept when finite and d2 < max_radius, ordered by (d2,
    index), the first k"""
    idx = np.full((len(queries), k), np.iinfo(np.uint64).max, dtype=np.uint64)
    d2 = np.full((len(queries), k), np.inf)
    cnt = np.zeros(len(queries), dtype=np.int32)
    ok_p = np.isfinite(points).all(axis=1)
    for q, qp in enumerate(queries):
        if not np.isfinite(qp).all():
            continue
        d = qp[None, :] - points
        dist = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        keep = np.nonzero(ok_p & (dist < max_radius))[0]
        order = keep[np.lexsort((keep, dist[keep]))][:k]
        cnt[q] = len(order)
        idx[q, :len(order)] = order
        d2[q, :len(order)] = dist[order]
    return idx, d2, cnt


def _clouds():
    rng = np.random.default_rng(7)
    yield "random", rng.uniform(-5, 5, (400, 3))
    az = rng.uniform(0, 2 * np.pi, 500)   # lidar-like: a ground ring and a wall, at map coordinates
    r = rng.uniform(2, 30, 500)
    pts = np.stack([r * np.cos(az), r * np.sin(az), rng.normal(0, 0.02, 500) - 1.7], 1) + [350.0, -120.0, 12.0]
    yield "lidar", pts
    base = rng.integers(-3, 3, (60, 3)).astype(float) * 0.5   # duplicates and equal distances everywhere
    yield "duplicates", base[rng.integers(0, 60, 300)]


@pytest.mark.parametrize("k", [1, 5, 10, 32])
def test_search_matches_numpy(k):
    for name, pts in _clouds():
        rng = np.random.default_rng(k)
        queries = np.concatenate([pts[rng.integers(0, len(pts), 40)] + rng.normal(0, 0.3, (40, 3)), pts[:10]])
        for max_radius in (DBL_MAX, 1.0, 0.05):
            got = orn.search(pts, queries, k, max_radius)
            ref = numpy_knn(pts, queries, k, max_radius)
            for g, r in zip(got, ref):
                np.testing.assert_array_equal(g, r, err_msg=f"{name} k={k} r={max_radius}")


def test_search_self_queries_and_non_finite():
    rng = np.random.default_rng(3)
    pts = rng.uniform(0, 1, (200, 3))
    pts[[5, 17]] = [np.nan, 0, 0], [0, np.inf, 0]
    got = orn.search(pts, None, 8)
    ref = numpy_knn(pts, pts, 8)
    for g, r in zip(got, ref):
        np.testing.assert_array_equal(g, r)
    assert got[2][5] == 0 and got[2][17] == 0                      # a non-finite query finds nothing
    assert not np.isin(got[0][got[0] != np.iinfo(np.uint64).max], [5, 17]).any()   # and is never found


def test_search_boundary_is_strict():
    pts = np.array([[0, 0, 0], [1, 0, 0], [0, 2, 0], [3, 0, 0.]])
    q = np.zeros((1, 3))
    idx, d2, cnt = orn.search(pts, q, 4, 1.0)      # d2 == max_radius is not kept
    assert cnt[0] == 1 and idx[0, 0] == 0
    idx, d2, cnt = orn.search(pts, q, 4, np.nextafter(1.0, 2.0))
    assert cnt[0] == 2 and list(idx[0, :2]) == [0, 1]
    for r in (0.0, -1.0):
        assert orn.search(pts, q, 4, r)[2][0] == 0
    ties = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0.]])
    idx, d2, cnt = orn.search(ties, q, 2)           # four equal d2: the two lowest indices
    assert list(idx[0]) == [0, 1] and cnt[0] == 2


@pytest.mark.parametrize("n", [0, 1, 3, 4])
def test_search_small_sets(n):
    pts = np.random.default_rng(n).uniform(0, 1, (n, 3))
    got = orn.search(pts, np.zeros((3, 3)), 5)
    ref = numpy_knn(pts, np.zeros((3, 3)), 5)
    for g, r in zip(got, ref):
        np.testing.assert_array_equal(g, r)
    assert (got[2] == n).all()


def _numpy_describe(pts):
    p = np.asarray(pts, dtype=np.float64)
    c = np.cov(p.T, bias=True)
    w, v = np.linalg.eigh(c)
    return w[::-1], v[:, ::-1], p.mean(0), c


def test_description_matches_numpy():
    rng = np.random.default_rng(11)
    for pts in (rng.normal(0, 1, (50, 3)) * [3, 1, 0.2], rng.uniform(-1, 1, (7, 3)),
                rng.normal(0, 1, (200, 3)) * [5, 0.1, 0.1] + [800.0, 300.0, 20.0]):
        d = orn.describe(pts)
        w, v, mean, cov = _numpy_describe(pts)
        np.testing.assert_allclose(d["barycenter"], mean, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(d["covariance"], cov[[0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]], rtol=1e-9, atol=1e-12)
        assert abs(abs(np.dot(d["normal"], v[:, 2])) - 1) < 1e-9 and abs(abs(np.dot(d["line"], v[:, 0])) - 1) < 1e-9
        np.testing.assert_allclose([d["linearity"], d["planarity"], d["a2D"]],
                                   [(w[0] - w[1]) / w[0], (w[1] - w[2]) / w[0],
                                    (np.sqrt(w[1]) - np.sqrt(w[2])) / np.sqrt(w[0])], rtol=1e-8, atol=1e-12)
        np.testing.assert_allclose(d["cov_det"], np.linalg.det(cov), rtol=1e-8, atol=1e-15)
        u = orn.describe(pts, centred=False)
        np.testing.assert_allclose(u["covariance"], d["covariance"], rtol=1e-6, atol=1e-9 * np.abs(pts).max() ** 2)


def test_classification_branches():
    rng = np.random.default_rng(5)
    g = np.arange(6) * 0.2
    plane = np.c_[np.repeat(g, 6), np.tile(g, 6), rng.normal(0, 1e-4, 36)]   # a square grid: planarity ~1
    line = np.c_[rng.uniform(-1, 1, 30), rng.normal(0, 1e-3, (30, 2))]
    blob = rng.normal(0, 1, (30, 3))
    ALL, T = abi.NB["ALL"], abi.NB_TYPE
    assert orn.describe(plane)["type"] == T["PLANAR"]
    assert orn.describe(line)["type"] == T["LINEAR"]
    assert orn.describe(blob)["type"] == T["NONE"]        # both computed, neither passes: NONE, never VOLUMIC
    # a is the linearity threshold, b the planarity threshold (the definition's names)
    assert orn.describe(line, linearity_threshold=0.9999999, planarity_threshold=0.0)["type"] == T["PLANAR"]
    assert orn.describe(line, linearity_threshold=0.5, planarity_threshold=1.0)["type"] == T["LINEAR"]
    cov_only = abi.NB["COV_DET"] | abi.NB["NORMAL"] | abi.NB["PLANARITY"]
    assert orn.describe(blob, values=cov_only)["type"] == T["VOLUMIC"]
    assert orn.describe(blob[:5], values=cov_only)["type"] == T["NONE"]    # VOLUMIC needs more than 5 points
    assert orn.describe(blob[:6], values=cov_only)["type"] == T["VOLUMIC"]
    assert orn.describe(blob, values=abi.NB["NORMAL"])["type"] == T["NONE"]
    small = orn.describe(blob[:4], values=ALL)                          # fewer than 5: defaults
    assert small["is_valid"] == 0 and small["type"] == T["NONE"] and small["planarity"] == -1 and small["a2D"] == -1
    assert not small["normal"].any() and not small["covariance"].any()
    sub = orn.describe(blob, values=abi.NB["LINE"])                    # fields not asked for keep their defaults
    assert sub["linearity"] == -1 and sub["cov_det"] == -1 and not sub["normal"].any() and sub["line"].any()
    same = orn.describe(np.tile([[1.0, 2.0, 3.0]], (6, 1)))            # coincident points: 0 / 0
    assert np.isnan(same["linearity"]) and np.isnan(same["planarity"]) and np.isnan(same["a2D"])
    assert same["type"] == T["NONE"] and same["is_valid"] == 1


def test_reference_unit_cases():
    rng = np.random.default_rng(1)
    for _ in range(2):   # test_neighborhood.cxx eigen / world_point: 1000 points in [-1, 1]^3, k 10 within d2 < 0.1
        pts = rng.uniform(-1, 1, (1000, 3))
        idx, d2, cnt = orn.search(pts, rng.uniform(-1, 1, (1, 3)), 10, 0.1)
        assert cnt[0] >= 1
    pts = rng.uniform(-1, 1, (10, 3))
    pts[:, 2] = 1.0          # normals: z = 1, ALL_BUT_KDTREE, |normal . z| == 1 exactly
    for centred in (True, False):
        d = orn.describe(pts, values=abi.NB["ALL_BUT_KDTREE"], centred=centred)
        assert abs(d["normal"][2]) == 1.0


def test_description_layout():
    eng = ct_icp_b200.engine()
    assert eng.fn("abi_sizeof")(b"cticp_neighborhood_description") == C.sizeof(abi.NeighborhoodDescription) == 160
    dt = abi.neighborhood_description_dtype()
    assert dt.itemsize == 160
    for name, _ in abi.NeighborhoodDescription._fields_:
        assert getattr(abi.NeighborhoodDescription, name).offset == dt.fields[name][1], name
    assert (abi.NB["ALL"], abi.NB["ALL_BUT_KDTREE"], abi.NB["A2D"], abi.NB_TYPE["VOLUMIC"]) == (127, 95, 64, 3)


def test_no_device_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    eng = ct_icp_b200.engine()
    with pytest.raises(ct_icp_b200.CticpError) as e:
        eng.neighborhood(np.zeros((10, 3)))
    assert e.value.code == abi.ERR_NO_DEVICE
    with pytest.raises(ct_icp_b200.CticpError) as e:
        eng.describe_point_sets(np.zeros((10, 3)))
    assert e.value.code == abi.ERR_NO_DEVICE
