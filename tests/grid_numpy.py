"""An independent NumPy statement of slam::SamplePointsInGrid under the engine's order contract (voxels in order of first
appearance, each voxel's points in input order) and its rejection rule: a lexsort on packed voxel keys. TEST
INFRASTRUCTURE."""
import numpy as np


def sample_points_in_grid(xyz, grid_size, num_points_per_voxel=1, max_num_points=-1):
    xyz = np.asarray(xyz, dtype=np.float64).reshape(-1, 3)
    with np.errstate(invalid="ignore", over="ignore"):
        q = xyz / grid_size
        ok = np.all(np.abs(q) < 2.0 ** 21, axis=1)
        k = np.zeros(q.shape, dtype=np.int64)
        k[ok] = np.trunc(q[ok]).astype(np.int64)
    ok &= np.all((k >= -(1 << 20)) & (k < (1 << 20)), axis=1)
    idx = np.nonzero(ok)[0]
    if len(idx) == 0:
        return np.zeros(0, dtype=np.uint64)
    kk = k[idx] + (1 << 20)
    keys = (kk[:, 0] << 42) | (kk[:, 1] << 21) | kk[:, 2]
    order = np.lexsort((idx, keys))
    sk, si = keys[order], idx[order]
    start = np.r_[True, sk[1:] != sk[:-1]]
    group = np.cumsum(start) - 1
    first = si[start][group]                       # each point's voxel's first index
    rank = np.arange(len(si)) - np.nonzero(start)[0][group]
    keep = rank < max(1, num_points_per_voxel)
    kept, kfirst = si[keep], first[keep]
    out = kept[np.lexsort((kept, kfirst))].astype(np.uint64)
    if max_num_points >= 0:
        out = out[:max_num_points + 1]
    return out
