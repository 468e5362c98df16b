"""The device voxel map at its edges, read from its snapshot bytes and compared with the NumPy model (voxel_map_model.py).

Every stored word is compared bit for bit: per voxel its key, count and the four fp32 words of every point, and per level
the header's capacity and counters. Where the data is dyadic (a 2^-6 grid, power-of-two resolutions) the oracle's export
must agree exactly too. The cases are the ones a rewrite of the commit or of the table rules gets wrong: long candidate
lists (the sorted path holds 512), voxel capacities 1 and 64, full voxels, the minimum-distance boundary, a second commit
round of every warp, growth and purges, eviction at exactly the distance, voxel normals and their per-point flips, the
21-bit coordinate range, and the odometry's fused and separate map updates.
"""
import ctypes as C
import struct

import numpy as np
import pytest

from ct_icp_b200 import _abi as abi
from ct_icp_b200 import synthetic as syn
from voxel_map_model import VoxelMapModel, pack_voxel

pytestmark = pytest.mark.gpu

HEADER = 72            # snapshot_format.h kHeaderBytes
SECTIONS = 5           # options, host state, trajectory, map, origins
DYADIC = 1.0 / 64
U = 2.0 ** -53
LO, HI = -(1 << 20), (1 << 20) - 1


# ---- the snapshot's map section (snapshot_format.h) ---------------------------------------------------------------------
class DevLevel:
    def __init__(self, header):
        self.header = header
        self.voxels = {}      # key -> (points (count, 4) f32, normal (4,) f64 or None)


def parse_map(blob):
    sizes = struct.unpack_from("<%dQ" % SECTIONS, blob, 16)
    offs = list(np.cumsum((HEADER,) + sizes[:-1]))
    at = int(offs[3]) + C.sizeof(abi.MapOptions)
    num_levels, has_normals, frame_count = struct.unpack_from("<IIQ", blob, at)
    at += 16
    levels = []
    for i in range(num_levels):
        cap, B, _, points, voxels, tombs, touched, overflow, records = struct.unpack_from("<QIIQIIIIQ", blob, at + 48 * i)
        levels.append((DevLevel(dict(cap=cap, B=B, points=points, voxels=voxels, tombs=tombs, touched=touched,
                                     overflow=overflow)), records))
    at += 48 * num_levels
    for L, records in levels:
        rec = np.frombuffer(blob, dtype=[("slot", "<u4"), ("count", "<u4"), ("key", "<u8")], count=records, offset=at)
        at += 16 * records
        npts = L.header["points"]
        pts = np.frombuffer(blob, dtype="<f4", count=4 * npts, offset=at).reshape(-1, 4)
        at += 16 * npts
        nrm = None
        if has_normals:
            nrm = np.frombuffer(blob, dtype="<f8", count=4 * records, offset=at).reshape(-1, 4)
            at += 32 * records
        cursor = 0
        for r, (slot, count, key) in enumerate(rec):
            if key == (1 << 64) - 2:
                continue
            assert int(key) not in L.voxels
            L.voxels[int(key)] = (pts[cursor:cursor + count], None if nrm is None else nrm[r])
            cursor += count
    origins = np.frombuffer(blob, dtype="<f8", count=3 * frame_count if has_normals else 0, offset=int(offs[4]))
    return dict(levels=[L for L, _ in levels], frame_count=frame_count, origins=origins.reshape(-1, 3),
                normals=bool(has_normals))


def assert_model(dev, model):
    """every level's header and every voxel's key, count and point words against the model; with normals the w sign
    is checked by assert_normals instead"""
    assert dev["frame_count"] == model.frame_count
    if model.normals:
        assert np.array_equal(dev["origins"], np.array(model.origins).reshape(-1, 3))
    for lvl, (D, L) in enumerate(zip(dev["levels"], model.levels)):
        assert D.header == L.header(), (lvl, D.header, L.header())
        assert set(D.voxels) == {pack_voxel(v) for v in L.voxels}, lvl
        for v, vox in L.voxels.items():
            got = D.voxels[pack_voxel(v)][0]
            want = vox.pts
            if model.normals:
                got, want = np.abs(got), np.abs(want)
            assert got.tobytes() == want.tobytes(), (lvl, v, got, want)


def assert_normals(dev, model):
    """the voxel normal against the model's fp64 eigenvector, within the Davis-Kahan bound of the one-pass moments
    (test_gpu_device_math.py's table: sin angle <= c u (lambda_1 + |mu|^2) / (lambda_2 - lambda_3), c = 64), and every
    point's flip against the begin position of its own frame"""
    checked = flips = 0
    for D, L in zip(dev["levels"], model.levels):
        for v, vox in L.voxels.items():
            pts, nrm = D.voxels[pack_voxel(v)]
            if vox.normal is None:
                assert nrm[3] == 0.0, v
                assert np.array_equal(np.sign(pts[:, 3]), np.ones(len(pts))), v
                continue
            assert nrm[3] == 1.0, v
            n = nrm[:3]
            lam = vox.eig
            mu = vox.pts[:, :3].astype(np.float64).mean(axis=0)
            gap = lam[1] - lam[0]
            bound = 64 * U * (lam[2] + mu @ mu) / gap if gap > 0 else np.inf
            if bound < 0.1:
                assert abs(np.linalg.norm(n) - 1.0) < 1e-12
                assert np.linalg.norm(np.cross(n, vox.normal)) <= bound + 1e-15, (v, n, vox.normal, bound)
                checked += 1
            for q in pts:
                f = int(abs(q[3])) - 1
                d = L.world(v, q) - dev["origins"][f]
                s = float(d @ n)
                if abs(s) > 1e-9 * (1.0 + np.linalg.norm(d)):
                    assert (q[3] < 0) == (s > 0), (v, q, s)
                    flips += 1
    return checked, flips


def assert_oracle(mo, me, levels=1):
    for lvl in range(levels):
        xo, vo = mo.export(lvl)
        xe, ve = me.export(lvl)
        assert np.array_equal(vo, ve) and np.array_equal(xo, xe)


def _map_options(b, res, B, md, cap=1024, normals=False, levels=None):
    o = b.legacy_map_options(res, B, md)
    if levels:
        o.num_resolutions = len(levels)
        for i, (r, bb, m) in enumerate(levels):
            o.resolutions[i].resolution, o.resolutions[i].max_num_points = r, bb
            o.resolutions[i].min_distance_between_points = m
    o.capacity_voxels = cap
    o.select_valid_normals_direction = 1 if normals else 0
    return o


def _maps(eng, orc, o, with_oracle=True):
    return eng.voxel_map(o), VoxelMapModel.from_options(o), (orc.voxel_map(o) if with_oracle else None)


def _insert(maps, pts, origin=None):
    me, model, mo = maps
    me.insert(pts, origin)
    model.insert(pts, origin)
    if mo is not None:
        mo.insert(pts, origin)


def _remove(maps, loc, dist):
    for m in maps:
        if m is not None:
            m.remove_far(loc, dist)


def _dyadic(p):
    return np.round(np.asarray(p) / DYADIC) * DYADIC


def _crowded(rng, counts, dyadic):
    """counts[k] candidates in voxel (k, k, 2k) of a 1 m grid plus a voxel of 50 exact duplicates, interleaved"""
    parts = []
    for k, n in enumerate(counts):
        parts.append(np.array([k, k, 2 * k], dtype=np.float64) + rng.uniform(0.0, 0.99, size=(n, 3)))
    parts.append(np.repeat([[-3.5, 7.25, 0.125]], 50, axis=0))
    p = np.concatenate(parts)
    p = p[rng.permutation(len(p))]
    return _dyadic(p) if dyadic else p


# ---- crowded voxels in one insert ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("min_dist", [0.0, 0.05, 0.25])
@pytest.mark.parametrize("B", [1, 20, 64])
def test_crowded_voxels(eng, orc, B, min_dist):
    rng = np.random.default_rng(100 * B + int(100 * min_dist))
    dyadic = min_dist != 0.05
    maps = _maps(eng, orc, _map_options(eng, 1.0, B, min_dist), with_oracle=dyadic)
    counts = [1, 31, 32, 33, 511, 512, 513, 4096]
    pts = _crowded(rng, counts, dyadic)
    _insert(maps, pts)
    me, model, mo = maps
    assert_model(parse_map(me.save()), model)
    if dyadic:
        assert_oracle(mo, me)
    assert len(model.levels[0].voxels[(-3, 7, 0)].pts) == 1     # exact duplicates: the first is accepted, the rest not
    # a second insert into the same, partly full voxels
    _insert(maps, _crowded(rng, counts[::-1], dyadic))
    assert_model(parse_map(me.save()), model)
    if dyadic:
        assert_oracle(mo, me)


def test_min_distance_boundary(eng, orc):
    maps = _maps(eng, orc, _map_options(eng, 1.0, 64, 0.25))
    base = np.array([0.5, 0.5, 0.5])
    at = [base + [0.25, 0, 0], base + [0, -0.25, 0], base + [0, 0, 0.25]]          # exactly min_dist: rejected
    beyond = [base + [-0.25 - DYADIC, 0, 0], base + [0, 0.25 + DYADIC, 0]]         # min_dist + 2^-6: accepted
    _insert(maps, np.array([base] + at + beyond))
    me, model, mo = maps
    assert model.levels[0].num_points == 3
    assert_model(parse_map(me.save()), model)
    assert_oracle(mo, me)
    xe, _ = me.export()
    assert np.array_equal(xe, np.array([base] + beyond))


# ---- commit rounds: a warp takes 32 voxels per round ----------------------------------------------------------------------
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_commit_rounds(eng, orc, delta):
    extra = 4000
    n_vox = 32 * 4 * 1056 + delta     # InsertDevice: warps_total = 4 · min(⌈n/4⌉, 1056) = 4224 for n >= 4224
    side = 52
    i = np.arange(n_vox)
    vox = np.stack([i % side, (i // side) % side, i // (side * side)], axis=1).astype(np.float64)
    rng = np.random.default_rng(7 + delta)
    pts = vox + _dyadic(rng.uniform(0.0, 0.99, size=(n_vox, 3)))
    more = vox[rng.integers(0, 64, size=extra)] + _dyadic(rng.uniform(0.0, 0.99, size=(extra, 3)))
    allp = np.concatenate([pts, more])
    allp = allp[rng.permutation(len(allp))]
    maps = _maps(eng, orc, _map_options(eng, 1.0, 6, 0.125), with_oracle=False)
    _insert(maps, allp)
    me, model, _ = maps
    dev = parse_map(me.save())
    assert dev["levels"][0].header["touched"] == n_vox
    assert_model(dev, model)
    _insert(maps, allp[::-3] + DYADIC)
    assert_model(parse_map(me.save()), model)


# ---- table maintenance ----------------------------------------------------------------------------------------------------
def _grid_points(rng, lo, hi, per_voxel):
    """per_voxel dyadic points in every voxel of the 1 m grid [lo, hi)^2 x {0}"""
    g = np.stack(np.meshgrid(np.arange(lo, hi), np.arange(lo, hi), [0], indexing="ij"), axis=-1).reshape(-1, 3)
    g = np.repeat(g.astype(np.float64), per_voxel, axis=0)
    u = _dyadic(rng.uniform(0.0, 0.99, size=g.shape))
    return np.where(g < 0, g - u, g + u)      # (int() truncates toward zero: voxel -k holds (-k - 1, -k])


def test_growth_purge_eviction(eng, orc):
    rng = np.random.default_rng(3)
    maps = _maps(eng, orc, _map_options(eng, 1.0, 8, 0.125, cap=1024))
    me, model, mo = maps
    L = model.levels[0]

    def check():
        assert_model(parse_map(me.save()), model)
        assert_oracle(mo, me)

    # exactly cap / 2 live voxels: no growth (the rule is a live load above 0.5)
    _insert(maps, _grid_points(rng, -16, 16, 1)[:512])
    check()
    assert L.cap == 1024 and L.num_voxels == 512
    # more voxels: the table doubles before the insert; three voxels at the eviction boundary of (0.5, 0.5, 0.5), 60.25:
    # A's first point is inside and its second outside, B's first outside and its second inside, C's first exactly at it
    special = np.array([[60.5, 0.5, 0.5], [-59.90625, 0.5, 0.5], [0.5, 60.75, 0.5],
                        [60.96875, 0.5, 0.5], [-59.5, 0.5, 0.5], [0.5, 60.5, 0.5]])
    _insert(maps, np.concatenate([special, _grid_points(rng, -40, 40, 1)]))
    check()
    cap = L.cap
    assert cap > 1024
    # eviction leaves a tombstone in its slot; only the first point decides, and `>` keeps C
    _remove(maps, (0.5, 0.5, 0.5), 60.25)
    check()
    assert (60, 0, 0) in L.voxels and (-59, 0, 0) not in L.voxels and (0, 60, 0) in L.voxels
    assert L.num_tombs == 1 and L.cap == cap
    # a purge at constant capacity once the tombstones pass a quarter of the table
    rebuilds = model.rebuilds
    _remove(maps, (0.5, 0.5, 0.5), 20.0)
    check()
    assert model.rebuilds == rebuilds + 1 and L.num_tombs == 0 and L.cap == cap
    # evicted voxels inserted again
    _insert(maps, _grid_points(rng, -40, 40, 2))
    check()


# ---- normals ----------------------------------------------------------------------------------------------------------------
def _plane_frame(rng, n_vox, per_voxel, tilt):
    """per_voxel points on a tilted plane in each of n_vox voxels along x"""
    x = np.repeat(np.arange(n_vox, dtype=np.float64), per_voxel) + rng.uniform(0.02, 0.98, n_vox * per_voxel)
    y = rng.uniform(0.02, 0.98, n_vox * per_voxel)
    z = 0.5 + tilt[0] * (x - np.floor(x) - 0.5) + tilt[1] * (y - 0.5) + rng.normal(0.0, 0.003, n_vox * per_voxel)
    return np.stack([x, y, z], axis=1)


def test_normals_and_flips(eng, orc):
    rng = np.random.default_rng(21)
    o = _map_options(eng, 1.0, 20, 0.02, cap=1024, normals=True)
    maps = _maps(eng, orc, o, with_oracle=False)
    me, model, _ = maps
    origins = [(0.0, 0.0, 10.0), (0.0, 0.0, -10.0), (30.0, 0.0, 10.0), (-5.0, 3.0, -8.0)]
    snaps = []
    for k in range(8):
        n_vox = 40 if k < 6 else 20            # the last frames touch only part of the voxels
        per = 2 if k < 4 else 5
        _insert(maps, _plane_frame(rng, n_vox, per, (0.2, -0.1)), origins[k % 4])
        dev = parse_map(me.save())
        assert_model(dev, model)
        checked, flips = assert_normals(dev, model)
        if k >= 2:
            assert checked >= 20 and flips > 100
        snaps.append(dev)
    # a voxel that got no point keeps its normal byte for byte; the full voxels took nothing
    last, prev = snaps[-1]["levels"][0].voxels, snaps[-2]["levels"][0].voxels
    for x in range(20, 40):
        key = pack_voxel((x, 0, 0))
        assert last[key][0].tobytes() == prev[key][0].tobytes()
        assert last[key][1].tobytes() == prev[key][1].tobytes()
    full = [v for v, vox in model.levels[0].voxels.items() if len(vox.pts) == 20]
    assert full
    before = parse_map(me.save())["levels"][0].voxels
    _insert(maps, _plane_frame(rng, 40, 6, (0.2, -0.1)), origins[0])
    after = parse_map(me.save())
    assert_model(after, model)
    assert_normals(after, model)
    for v in full:
        key = pack_voxel(v)
        assert after["levels"][0].voxels[key][0].tobytes() == before[key][0].tobytes()
        assert after["levels"][0].voxels[key][1].tobytes() == before[key][1].tobytes()
    # normals survive growth and purges, byte for byte
    keep = parse_map(me.save())["levels"][0].voxels
    cap = model.levels[0].cap
    far = _plane_frame(rng, 1200, 1, (0.0, 0.0)) + np.array([0.0, 50.0, 0.0])
    _insert(maps, far, origins[1])
    assert model.levels[0].cap > cap
    _remove(maps, (20.0, 0.5, 0.5), 30.0)
    assert model.levels[0].num_tombs == 0
    dev = parse_map(me.save())
    assert_model(dev, model)
    assert_normals(dev, model)
    for key, (pts, nrm) in keep.items():
        assert dev["levels"][0].voxels[key][0].tobytes() == pts.tobytes()
        assert dev["levels"][0].voxels[key][1].tobytes() == nrm.tobytes()


# ---- the coordinate range ---------------------------------------------------------------------------------------------------
def test_coordinate_range(eng, orc):
    res = 0.5
    o = _map_options(eng, res, 20, 0.0, cap=1024)
    o.default_radius = 1.0            # a 5^3 stencil
    maps = _maps(eng, orc, o)
    me, model, mo = maps

    def at(vx, vy, vz, off=(0.25, 0.125, 0.375)):
        return [c * res + (f if c >= 0 else -f) for c, f in zip((vx, vy, vz), off)]

    inside = np.array([at(LO, 0, 0), at(HI, 0, 0), at(0, LO, 0), at(0, HI, 0), at(0, 0, LO), at(0, 0, HI),
                       at(LO, LO, LO), at(HI, HI, HI), at(3, 4, 5), at(-2, 0, 1)])
    _insert(maps, inside)
    assert_model(parse_map(me.save()), model)
    assert_oracle(mo, me)
    xe, ve = me.export()
    assert len(xe) == len(inside)
    # out of range: a voxel 2^20 or -2^20 - 1 on any axis, the voxel whose key would be kEmptyKey, huge and non-finite
    outside = np.array([at(HI + 1, 0, 0), at(LO - 1, 0, 0), at(0, 4, HI + 1), at(0, LO - 1, 7), at(LO - 1, LO - 1, LO - 1),
                        at(5, 5, HI + 3), [1e300, 0, 0], [0, -1e20, 0], [np.nan, 0, 0], [0, 0, np.inf]])
    before = me.save()
    me.insert(outside)
    model.insert(outside)
    dev = parse_map(me.save())
    assert_model(dev, model)
    assert dev["levels"][0].header["touched"] == 0
    ba, bb = parse_map(before)["levels"][0].voxels, dev["levels"][0].voxels
    assert {k: v[0].tobytes() for k, v in ba.items()} == {k: v[0].tobytes() for k, v in bb.items()}
    assert_oracle(mo, me)
    mixed = np.concatenate([outside, np.array([at(1, 1, 1)])])
    _insert(maps, mixed[-1:])
    me.insert(mixed[:-1])
    model.insert(mixed[:-1])
    assert_model(parse_map(me.save()), model)
    assert_oracle(mo, me)
    # a query whose voxel is out of range finds none of the points of the voxel its key would alias: (2^20, 0, 0) aliases
    # (-2^20, 0, 0), whose point reads back 0.3 m from the query, (0, 4, 2^20) aliases (0, 5, -2^20)
    _insert(maps, np.array([at(0, 5, LO)]))
    q = np.array([[(HI + 1) * res + 0.05, 0.125, 0.375], at(LO - 1, 0, 0), [0.125, 4 * res + 0.125, (HI + 1) * res + 0.01],
                  [2e9 * res, 0, 0], [-3e12, 0, 0], at(HI, 0, 0)])
    for _, cnt in (me.compute_neighborhoods(q, 20), me.radius_search(q, 1.0, 20)):
        assert np.array_equal(cnt, np.zeros(len(q)))
    # queries whose stencil stays inside the range find the edge voxels (the oracle's search cannot be asked: the
    # reference walks the stencil with `short` loop variables, map.h:470-472)
    q_in = np.array([at(HI - 2, 0, 0, (0.45, 0.125, 0.375)), at(LO + 2, 0, 0, (0.45, 0.125, 0.375))])
    pe, ce = me.compute_neighborhoods(q_in, 20)
    assert np.array_equal(ce, [1, 1])
    xe, ve = me.export()
    for k, v in enumerate(((HI, 0, 0), (LO, 0, 0))):
        assert np.array_equal(pe[k, 0], xe[np.all(ve == v, axis=1)][0])


# ---- the odometry's map update ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dense_seq():
    return syn.make_sequence(5, syn.HDL64, seed=77)


def _odometry_maps(eng, seq, monkeypatch, fused, ctas):
    monkeypatch.setenv("CTICP_FUSED_MAP_UPDATE", str(fused))
    monkeypatch.setenv("CTICP_UPDATE_CTAS_PER_SM", str(ctas))
    o = eng.default_odometry_options()
    o.ct_icp_options.solver = abi.SOLVER["GN"]
    o.ct_icp_options.num_iters_icp = 4
    o.ct_icp_options.min_number_neighbors = 10
    o.map_options = eng.legacy_map_options(0.2, 20, 0.05)
    o.voxel_size, o.sample_voxel_size, o.max_distance = 0.1, 1.5, 60.0
    o.init_num_frames = 3
    o.debug_print = 0
    o.ct_icp_options.debug_print = 0
    od = eng.odometry(o)
    out = []
    for s in seq:
        sm = od.RegisterFrame(s["xyz"], s["t"], s["frame_idx"])
        assert sm.success
        dev = parse_map(od.save())
        out.append(({k: (v[0].tobytes(), None if v[1] is None else v[1].tobytes()) for k, v in dev["levels"][0].voxels.items()},
                    {k: dev["levels"][0].header[k] for k in ("cap", "points", "voxels", "tombs", "overflow")},
                    dev["levels"][0].header["touched"]))
    od.close()
    return out


def test_fused_and_separate_map_updates_agree(eng, dense_seq, monkeypatch):
    runs = {(f, c): _odometry_maps(eng, dense_seq, monkeypatch, f, c) for f, c in ((1, 4), (1, 1), (0, 4), (0, 1))}
    ref = runs[(1, 4)]
    # the fused grid at one CTA per SM has 132 · 4 warps: some frame touches more than 32 voxels per warp
    assert max(t for _, _, t in ref) > 32 * 4 * 132
    for key, run in runs.items():
        for frame, (a, b) in enumerate(zip(ref, run)):
            assert a[1] == b[1], (key, frame, a[1], b[1])
            assert a[0] == b[0], (key, frame)
