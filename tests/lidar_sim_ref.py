"""A NumPy restatement of the spinning-LiDAR sweeps of include/cticp.h ("Spinning-LiDAR sweeps"), for the tests: ray order,
column timestamps, sensor directions from the host C library (through ctypes), the engine's quaternion rotation operation
for operation, then tools/raycast.c (the host caster) for the ranges and the keep rule. The caller supplies each column's
pose, so the same restatement checks the device against its own trajectory lookups and against synthetic.generate_scan's
analytic poses."""
import ctypes
import ctypes.util
import math

import numpy as np

from ct_icp_b200 import synthetic

_LIBM = None


def libm():
    global _LIBM
    if _LIBM is None:
        _LIBM = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
        for name in ("cos", "sin"):
            getattr(_LIBM, name).restype = ctypes.c_double
            getattr(_LIBM, name).argtypes = [ctypes.c_double]
    return _LIBM


def elevations(sensor):
    """the ring elevations in degrees, top to bottom: the explicit table, else generate_scan's np.linspace"""
    if getattr(sensor, "elev_table_deg", None) is not None:
        return np.asarray(sensor.elev_table_deg, dtype=np.float64)
    return np.linspace(sensor.elev_max_deg, sensor.elev_min_deg, sensor.n_rings)


def sensor_directions(sensor):
    """(n_rings n_azimuth, 3) directions in the sensor frame, ray i = ring n_azimuth + j"""
    m = libm()
    el = [float(e) * (math.pi / 180.0) for e in elevations(sensor)]
    naz = sensor.n_azimuth
    az = [-2.0 * math.pi * j / naz for j in range(naz)]
    cel = np.array([m.cos(e) for e in el])
    sel = np.array([m.sin(e) for e in el])
    caz = np.array([m.cos(a) for a in az])
    saz = np.array([m.sin(a) for a in az])
    d = np.empty((len(el), naz, 3))
    d[..., 0] = cel[:, None] * caz[None, :]
    d[..., 1] = cel[:, None] * saz[None, :]
    d[..., 2] = sel[:, None]
    return d.reshape(-1, 3)


def column_times(t0, sensor):
    return t0 + ((np.arange(sensor.n_azimuth) + 0.5) / sensor.n_azimuth) * sensor.period


def qnormalized(q):
    n = np.sqrt(((q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]) + q[:, 2] * q[:, 2]) + q[:, 3] * q[:, 3])
    return q / n[:, None]


def qrot(q, v):
    """Eigen's _transformVector (se3.cuh qrot): uv = 2 (q.vec x v); (v + w uv) + q.vec x uv, row by row"""
    x, y, z, w = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    uv = np.stack([y * v[:, 2] - z * v[:, 1], z * v[:, 0] - x * v[:, 2], x * v[:, 1] - y * v[:, 0]], -1)
    uv = uv + uv
    c = np.stack([y * uv[:, 2] - z * uv[:, 1], z * uv[:, 0] - x * uv[:, 2], x * uv[:, 1] - y * uv[:, 0]], -1)
    return (v + w[:, None] * uv) + c


def raycast(boxes, cyl, o, d, max_range, key):
    """tools/raycast.c (always with the ground plane) under the per-call key"""
    o = np.ascontiguousarray(o, dtype=np.float64)
    d = np.ascontiguousarray(d, dtype=np.float64)
    boxes = np.ascontiguousarray(boxes, dtype=np.float64).reshape(-1, 7)
    cyl = np.ascontiguousarray(cyl, dtype=np.float64).reshape(-1, 4)
    out = np.empty(len(o))
    synthetic._raycast_lib().raycast_scene(o.ctypes.data, d.ctypes.data, len(o), boxes.ctypes.data, len(boxes),
                                           cyl.ctypes.data, len(cyl), float(max_range), key & 0xFFFFFFFFFFFFFFFF,
                                           out.ctypes.data)
    return out


def sweep(boxes, cyl, sensor, t0, frame_id, seed, quat, tr, ds=None):
    """One sweep with noise_sigma 0 from the columns' poses (quat (n_azimuth, 4) x y z w, tr (n_azimuth, 3)). Returns a
    dict: ray_index, range r and t of the kept rays, raw and world xyz in fp64, and every ray's range (all_r)."""
    ds = sensor_directions(sensor) if ds is None else ds
    naz = sensor.n_azimuth
    j = np.tile(np.arange(naz), sensor.n_rings)
    q = qnormalized(np.asarray(quat, dtype=np.float64))[j]
    o = np.asarray(tr, dtype=np.float64)[j]
    dw = qrot(q, ds)
    r = raycast(boxes, cyl, o, dw, sensor.max_range, (seed * 1000003 + frame_id) & 0xFFFFFFFFFFFFFFFF)
    keep = np.isfinite(r) & (r > sensor.min_range) & (r < sensor.max_range)
    idx = np.nonzero(keep)[0]
    rk = r[idx]
    return {"ray_index": idx, "r": rk, "t": column_times(t0, sensor)[j[idx]], "raw": ds[idx] * rk[:, None],
            "world": o[idx] + dw[idx] * rk[:, None], "all_r": r, "dw": dw, "o": o}


def trajectory_poses(traj, t_end, rate=100.0):
    """abi.Pose samples of a synthetic.Trajectory every 1 / rate seconds over [0, t_end] (frame id 0, by timestamp)"""
    from scipy.spatial.transform import Rotation
    from ct_icp_b200 import _abi as abi
    ts = np.arange(int(math.ceil(t_end * rate)) + 2) / rate
    quat = Rotation.from_matrix(traj.rotation(ts)).as_quat()
    pos = traj.position(ts)
    return [abi.Pose.make(quat[k].tolist(), pos[k].tolist(), float(ts[k]), 0) for k in range(len(ts))]


def device_columns(trajectory, sensor, t0):
    """the columns' poses as cticp_trajectory_interpolate gives them: (quat, tr)"""
    p = trajectory.interpolate(column_times(t0, sensor))
    return np.asarray(p["quat"], dtype=np.float64), np.asarray(p["tr"], dtype=np.float64)
