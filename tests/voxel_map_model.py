"""A plain NumPy model of the device voxel map (device_map.cu / device_map.cuh) over what the device stores.

It restates InsertPointCloud, RemoveElementsFarFromLocation (include/ct_icp/map.h:153-322) and the table rules of
DeviceMap (EnsureRoomFor, MaintainTables), one voxel at a time and in input order:

- a point's voxel is voxel_coord_rcp's integer, int(p / res) truncated toward zero; a point that is non-finite or whose
  voxel coordinate lies outside [-2^20, 2^20) on any axis is skipped (the 21-bit keys cannot hold it);
- the stored point is float32(world - voxel * res), with w = +-(source frame ordinal + 1);
- a candidate is rejected when !(d2 > min_dist^2) against any stored offset, d2 taken in fp64 between the candidate's
  fp64 offset and the stored fp32 offsets, candidates in ascending input index; a voxel at max_num_points takes none,
  and the first point of a new voxel is always accepted;
- a voxel is evicted when its FIRST stored point is farther than the distance (`>`);
- a voxel that received a point and holds >= 5 gets the normal of all its points, and every point's sign says whether
  its copy of the normal is flipped against the begin position of the frame it came from.

The map is keyed by voxel, not by slot: which slot a voxel lands in depends on the order in which claims arrive.
Normals are the fp64 eigenvector of the smallest eigenvalue; their sign is arbitrary, so `flip` is recorded against the
model's own normal and a comparison aligns the two signs first.
"""
import math

import numpy as np

VOXEL_BIAS = 1 << 20
COORD_LIMIT = float(1 << 21)
MAX_B = 64


def next_pow2(v):
    p = 1
    while p < v:
        p <<= 1
    return p


def voxel_coord(p, res):
    """voxel_coord_rcp (device_map.cuh): int(p / res), toward zero. The device's reciprocal product agrees with the
    quotient except within ~1e-15 of an integer, where it divides."""
    return int(p / res)


def voxel_of(p, res):
    """The voxel of a world point, or None when the map skips it (voxel_key, device_map.cuh)."""
    inv = 1.0 / res
    if not all(abs(c * inv) < COORD_LIMIT for c in p):     # (NaN and inf fail too)
        return None
    v = tuple(voxel_coord(c, res) for c in p)
    if not all(-VOXEL_BIAS <= c < VOXEL_BIAS for c in v):
        return None
    return v


def pack_voxel(v):
    x, y, z = (c + VOXEL_BIAS for c in v)
    return (x << 42) | (y << 21) | z


def unpack_voxel(key):
    return ((key >> 42) & 0x1FFFFF) - VOXEL_BIAS, ((key >> 21) & 0x1FFFFF) - VOXEL_BIAS, (key & 0x1FFFFF) - VOXEL_BIAS


def voxel_normal(offsets):
    """fp64 normal of a voxel's points (eigenvector of the smallest eigenvalue of their covariance) and the eigenvalues,
    ascending."""
    q = np.asarray(offsets, dtype=np.float64)
    c = np.cov(q.T, bias=True)
    lam, vec = np.linalg.eigh(c)
    return vec[:, 0], lam


class Voxel:
    __slots__ = ("pts", "normal", "eig")

    def __init__(self):
        self.pts = np.zeros((0, 4), dtype=np.float32)   # x, y, z offset from the voxel origin, w = +-(ordinal + 1)
        self.normal = None                              # the model's normal once computed (fp64)
        self.eig = None


class Level:
    def __init__(self, res, max_num_points, min_dist, cap):
        self.res, self.B, self.min_dist = float(res), int(max_num_points), float(min_dist)
        self.min_dist2 = self.min_dist * self.min_dist
        self.cap = cap
        self.voxels = {}
        self.num_points = 0
        self.num_tombs = 0
        self.num_touched = 0
        self.overflow = 0

    @property
    def num_voxels(self):
        return len(self.voxels)

    def header(self):
        """What the snapshot's level header holds."""
        return dict(cap=self.cap, B=self.B, points=self.num_points, voxels=self.num_voxels, tombs=self.num_tombs,
                    touched=self.num_touched, overflow=self.overflow)

    def world(self, v, q):
        """fp64 world position of a stored point."""
        return np.array([v[0] * self.res + float(q[0]), v[1] * self.res + float(q[1]), v[2] * self.res + float(q[2])])


class VoxelMapModel:
    """levels: [(resolution, max_num_points, min_distance_between_points)]; capacity_voxels as cticp_map_options."""

    def __init__(self, levels, capacity_voxels=0, normals=False):
        self.levels = []
        for res, B, md in levels:
            if not 1 <= B <= MAX_B:
                raise ValueError("max_num_points out of 1..64")
            cap = capacity_voxels if capacity_voxels else ((1 << 20) if res < 0.5 else (1 << 18))
            self.levels.append(Level(res, B, md, next_pow2(max(cap, 1024))))
        self.normals = normals
        self.origins = []      # begin position of every inserted frame
        self.frame_count = 0
        self.rebuilds = 0

    @classmethod
    def from_options(cls, o):
        """From a cticp_map_options (abi.MapOptions)."""
        levels = [(o.resolutions[i].resolution, o.resolutions[i].max_num_points,
                   o.resolutions[i].min_distance_between_points) for i in range(o.num_resolutions)]
        return cls(levels, o.capacity_voxels, bool(o.select_valid_normals_direction))

    # ---- the tables ---------------------------------------------------------------------------------------------------
    def _rebuild(self, L, cap):
        L.cap = cap
        L.num_tombs = 0
        L.overflow = 0
        self.rebuilds += 1

    def ensure_room_for(self, n_new):
        """EnsureRoomFor: before an insert of n_new points, every one of which may open a voxel."""
        for L in self.levels:
            live = L.num_voxels + n_new
            used = live + L.num_tombs
            if used * 10 <= L.cap * 8:
                continue
            cap = L.cap
            while live * 2 > cap:
                cap *= 2
            self._rebuild(L, cap)

    def maintain_tables(self):
        """MaintainTables: grow when the live load passes 0.5, purge tombstones when the used load passes 0.7 or the
        tombstones a quarter of the table."""
        for L in self.levels:
            used = L.num_voxels + L.num_tombs
            grow = L.num_voxels * 2 > L.cap
            purge = used * 10 > L.cap * 7 or L.num_tombs * 4 > L.cap
            if grow or purge:
                self._rebuild(L, L.cap * 2 if grow else L.cap)

    # ---- the operations -----------------------------------------------------------------------------------------------
    def insert(self, xyz, origin=None):
        """cticp_map_insert_from: EnsureRoomFor, the insert on every level, MaintainTables."""
        xyz = np.asarray(xyz, dtype=np.float64).reshape(-1, 3)
        if len(xyz) == 0:
            return
        self.ensure_room_for(len(xyz))
        ordinal = self.frame_count
        self.frame_count += 1
        if self.normals:
            self.origins.append(np.zeros(3) if origin is None else np.asarray(origin, dtype=np.float64))
        for L in self.levels:
            self._insert_level(L, xyz, ordinal)
        self.maintain_tables()

    def _insert_level(self, L, xyz, ordinal):
        cands = {}
        for i, p in enumerate(xyz):
            v = voxel_of(p, L.res)
            if v is not None:
                cands.setdefault(v, []).append(i)
        L.num_touched = len(cands)
        for v, idx in cands.items():
            vox = L.voxels.get(v)
            if vox is None:
                vox = L.voxels[v] = Voxel()
            count0 = len(vox.pts)
            if count0 >= L.B:
                continue
            o = np.array([v[0] * L.res, v[1] * L.res, v[2] * L.res])
            pts = [tuple(q) for q in vox.pts]
            for i in idx:                                          # ascending input index
                if len(pts) >= L.B:
                    break
                l = xyz[i] - o                                     # fp64 offset of the candidate
                reject = False
                for q in pts:
                    dx, dy, dz = float(q[0]) - l[0], float(q[1]) - l[1], float(q[2]) - l[2]
                    if not (dx * dx + dy * dy + dz * dz > L.min_dist2):
                        reject = True
                        break
                if not reject:
                    pts.append((np.float32(l[0]), np.float32(l[1]), np.float32(l[2]), np.float32(ordinal + 1)))
            vox.pts = np.array(pts, dtype=np.float32).reshape(-1, 4)
            L.num_points += len(pts) - count0
            if self.normals and len(pts) > count0 and len(pts) >= 5:
                self._orient(L, v, vox)

    def _orient(self, L, v, vox):
        n, lam = voxel_normal(vox.pts[:, :3].astype(np.float64))
        vox.normal, vox.eig = n, lam
        for j, q in enumerate(vox.pts):
            f = int(abs(q[3])) - 1
            d = L.world(v, q) - self.origins[f]
            flip = float(d @ n) > 0.0
            vox.pts[j, 3] = -abs(q[3]) if flip else abs(q[3])

    def remove_far(self, location, distance):
        """RemoveElementsFarFromLocation, then MaintainTables: a voxel goes when its first point is farther than
        `distance` (the device leaves a tombstone in its slot)."""
        loc = np.asarray(location, dtype=np.float64)
        for L in self.levels:
            gone = []
            for v, vox in L.voxels.items():
                d = L.world(v, vox.pts[0]) - loc
                if math.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]) > distance:
                    gone.append(v)
            for v in gone:
                L.num_points -= len(L.voxels.pop(v).pts)
                L.num_tombs += 1
        self.maintain_tables()

    def clear(self):
        for L in self.levels:
            L.voxels.clear()
            L.num_points = L.num_tombs = L.num_touched = L.overflow = 0
        self.origins = []
        self.frame_count = 0

    # ---- views --------------------------------------------------------------------------------------------------------
    def export(self, level=0):
        """GetMapPoints in (voxel, insertion) order: (fp64 world xyz (P, 3), voxel (P, 3) int32), as VoxelMap.export."""
        L = self.levels[level]
        xyz, vox = [], []
        for v in sorted(L.voxels):
            for q in L.voxels[v].pts:
                xyz.append(L.world(v, q))
                vox.append(v)
        return (np.array(xyz, dtype=np.float64).reshape(-1, 3), np.array(vox, dtype=np.int32).reshape(-1, 3))
