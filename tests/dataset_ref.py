"""NumPy restatement of the dataset readers the GPU tests compare against (include/cticp.h, "Dataset sequences"):
NCLTIterator::NextBatch / DoNext over velodyne_hits.bin bytes, kitti_frame_filter, and the writers of the file formats
(velodyne_hits.bin packets, binary PLY, KITTI / NCLT / HILTI ground truth) the tests build their fixtures with."""
import math
import struct

import numpy as np

MAGIC = 44444
HEADER = struct.Struct("<4HIQI")   # magic x4, num_hits, utime (byte 12), padding
HIT = np.dtype([("x", "<u2"), ("y", "<u2"), ("z", "<u2"), ("i", "u1"), ("l", "u1")])


# ---- NCLT ------------------------------------------------------------------------------------------------------------
def quantise(xyz):
    """metres → the u16 counts of a hit: round((v + 100) / 0.005), clipped to [0, 65535]"""
    return np.clip(np.rint((np.asarray(xyz, dtype=np.float64) + 100.0) / 0.005), 0, 65535).astype(np.uint16)


def pack_packet(utime, q, intensity=None, laser=None):
    """one packet: the 24-byte header and len(q) hits (q: (k, 3) uint16)"""
    q = np.asarray(q, dtype=np.uint16).reshape(-1, 3)
    hits = np.zeros(len(q), dtype=HIT)
    hits["x"], hits["y"], hits["z"] = q[:, 0], q[:, 1], q[:, 2]
    hits["i"] = 0 if intensity is None else intensity
    hits["l"] = np.arange(len(q)) % 32 if laser is None else laser
    return HEADER.pack(MAGIC, MAGIC, MAGIC, MAGIC, len(q), int(utime), 0) + hits.tobytes()


def walk(data):
    """the reference's sequential read: [(offset, num_hits, utime)], the offset where it stopped and why
    ('end', 'truncated' or 'bad_magic')"""
    data = bytes(data)
    n, off, out = len(data), 0, []
    while off < n:
        if n - off >= 8 and struct.unpack_from("<4H", data, off) != (MAGIC,) * 4:
            return out, off, "bad_magic"
        if n - off < HEADER.size:
            return out, off, "truncated"
        _, _, _, _, nh, ut, _ = HEADER.unpack_from(data, off)
        end = off + HEADER.size + 8 * nh
        if end > n:
            return out, off, "truncated"
        out.append((off, nh, ut))
        off = end
    return out, off, "end"


def decode(data, num_aggregated=220, final=True):
    """DoNext over the bytes: a dict with frames [(xyz (n, 3) float64, t (n,) float64)], info [(n, t_first, t_max)],
    num_packets and bytes_used; raises ValueError where the engine refuses"""
    data = bytes(data)
    packets, off, why = walk(data)
    if why == "bad_magic":
        raise ValueError("bad magic at %d" % off)
    if final and why == "truncated":
        raise ValueError("truncated at %d" % off)
    A = num_aggregated
    nf = (len(packets) + A - 1) // A if final else len(packets) // A
    packets = packets[:nf * A]
    frames, info = [], []
    for f in range(nf):
        xs, ts = [], []
        for (o, nh, ut) in packets[f * A:(f + 1) * A]:
            h = np.frombuffer(data, dtype=HIT, count=nh, offset=o + HEADER.size)
            q = np.stack([h["x"], h["y"], h["z"]], 1).astype(np.float64)
            xs.append(q * 0.005 - 100.0)
            ts.append(np.full(nh, float(ut)))
        xyz = np.concatenate(xs) if xs else np.zeros((0, 3))
        t = np.concatenate(ts) if ts else np.zeros(0)
        frames.append((xyz, t))
        info.append((len(t), t[0] if len(t) else np.nan, t.max() if len(t) else np.nan))
    used = packets[-1][0] + HEADER.size + 8 * packets[-1][1] if packets else 0
    return {"frames": frames, "info": info, "num_packets": len(packets), "bytes_used": used}


# ---- KITTI filter ------------------------------------------------------------------------------------------------------
def kitti_frame_filter(xyz):
    """kitti_frame_filter (dataset.cpp:85-110) of (n, 3) float64 points, Eigen's operations in Eigen's order"""
    p = np.asarray(xyz, dtype=np.float64)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    angle = 0.205 * math.pi / 180.0
    sa, ca = math.sin(angle), math.cos(angle)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        ux, uy, uz = 0.0, 0.0, 1.0
        ax, ay, az = y * uz - z * uy, z * ux - x * uz, x * uy - y * ux
        sq = (ax * ax + ay * ay) + az * az
        s = np.sqrt(np.where(sq > 0, sq, 1.0))
        ax, ay, az = np.where(sq > 0, ax / s, ax), np.where(sq > 0, ay / s, ay), np.where(sq > 0, az / s, az)
        sx, sy, sz = sa * ax, sa * ay, sa * az
        cx, cy, cz = (1.0 - ca) * ax, (1.0 - ca) * ay, (1.0 - ca) * az
        tmp = cx * ay
        r01, r10 = tmp - sz, tmp + sz
        tmp = cx * az
        r02, r20 = tmp + sy, tmp - sy
        tmp = cy * az
        r12, r21 = tmp - sx, tmp + sx
        r00, r11, r22 = cx * ax + ca, cy * ay + ca, cz * az + ca
        out = np.stack([(r00 * x + r01 * y) + r02 * z, (r10 * x + r11 * y) + r12 * z, (r20 * x + r21 * y) + r22 * z], 1)
    keep = z > -5.0
    return np.where(keep[:, None], out, 0.0)


# ---- PLY ------------------------------------------------------------------------------------------------------------
PLY_TYPES = {"float32": "float", "float64": "double", "uint8": "uchar", "int8": "char", "uint16": "ushort",
             "int16": "short", "uint32": "uint", "int32": "int"}


def ply_bytes(records):
    """a binary_little_endian PLY file of a structured array's fields, in order, as one packed vertex element"""
    dt = records.dtype
    lines = ["ply", "format binary_little_endian 1.0", "comment written by the dataset tests",
             "element vertex %d" % len(records)]
    for name in dt.names:
        lines.append("property %s %s" % (PLY_TYPES[dt.fields[name][0].name], name))
    lines.append("end_header")
    packed = np.zeros(len(records), dtype=[(n, dt.fields[n][0].newbyteorder("<")) for n in dt.names])
    for n in dt.names:
        packed[n] = records[n]
    return ("\n".join(lines) + "\n").encode() + packed.tobytes()


# ---- ground truth ----------------------------------------------------------------------------------------------------
def quat_to_matrix(q):   # (x, y, z, w), unit
    from scipy.spatial.transform import Rotation
    return Rotation.from_quat(q).as_matrix()


def matrix_to_quat(R):
    from scipy.spatial.transform import Rotation
    return Rotation.from_matrix(R).as_quat()


def se3(q, t):
    M = np.eye(4)
    M[:3, :3] = quat_to_matrix(np.asarray(q) / np.linalg.norm(q))
    M[:3, 3] = t
    return M


KITTI_CALIB = [
    (np.array([[4.276802385584e-04, -9.999672484946e-01, -8.084491683471e-03],
               [-7.210626507497e-03, 8.081198471645e-03, -9.999413164504e-01],
               [9.999738645903e-01, 4.859485810390e-04, -7.206933692422e-03]]),
     np.array([-1.198459927713e-02, -5.403984729748e-02, -2.921968648686e-01])),
    (np.array([[2.347736981471e-04, -9.999441545438e-01, -1.056347781105e-02],
               [1.044940741659e-02, 1.056535364138e-02, -9.998895741176e-01],
               [9.999453885620e-01, 1.243653783865e-04, 1.045130299567e-02]]),
     np.array([-2.796816941295e-03, -7.510879138296e-02, -2.721327964059e-01])),
    (np.array([[-1.857739385241e-03, -9.999659513510e-01, -8.039975204516e-03],
               [-6.481465826011e-03, 8.051860151134e-03, -9.999466081774e-01],
               [9.999773098287e-01, -1.805528627661e-03, -6.496203536139e-03]]),
     np.array([-4.784029760483e-03, -7.337429464231e-02, -3.339968064433e-01]))]
KITTI360_CALIB = (np.array([[9.999290633685804508e-01, 5.805355888196038310e-03, 1.040029024212630118e-02],
                            [5.774300279226996999e-03, -9.999787876452227442e-01, 3.013573682642321436e-03],
                            [1.041756443854582707e-02, -2.953305511449066945e-03, -9.999413744330052367e-01]]),
                  np.array([-7.640302229235816922e-01, 2.966030253893782165e-01, -8.433819635885287935e-01]))


def ypr_matrix(yaw, pitch, roll):
    from scipy.spatial.transform import Rotation
    return Rotation.from_euler("ZYX", [yaw, pitch, roll]).as_matrix()


def nclt_calib():
    M = np.eye(4)
    M[:3, :3] = ypr_matrix(-90.703 / 180 * math.pi, 0.166 / 180 * math.pi, 0.807 / 180 * math.pi)
    M[:3, 3] = (0.002, -0.004, -0.957)
    return M


def eigen_quat(R):
    """Eigen's Quaternion(Matrix3) (the trace-based construction, not a projection onto the rotations): (x, y, z, w)"""
    R = np.asarray(R, dtype=np.float64)
    t = R[0, 0] + R[1, 1] + R[2, 2]
    if t > 0:
        t = math.sqrt(t + 1.0)
        w = 0.5 * t
        t = 0.5 / t
        return np.array([(R[2, 1] - R[1, 2]) * t, (R[0, 2] - R[2, 0]) * t, (R[1, 0] - R[0, 1]) * t, w])
    i = 0
    if R[1, 1] > R[0, 0]:
        i = 1
    if R[2, 2] > R[i, i]:
        i = 2
    j, k = (i + 1) % 3, (i + 2) % 3
    t = math.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0)
    c = [0.0, 0.0, 0.0]
    c[i] = 0.5 * t
    t = 0.5 / t
    w = (R[k, j] - R[j, k]) * t
    c[j] = (R[j, i] + R[i, j]) * t
    c[k] = (R[k, i] + R[i, k]) * t
    return np.array(c + [w])


def calib_matrix(dataset, sequence_id=0):
    """the Calib of transform_poses: the pose in the LiDAR frame is CalibI · M · Calib"""
    if dataset in ("KITTI", "KITTI_raw"):
        R, t = KITTI_CALIB[0 if sequence_id <= 2 else 1 if sequence_id == 3 else 2]
        return se3(eigen_quat(R), t)
    if dataset == "KITTI_360":
        return se3(eigen_quat(KITTI360_CALIB[0]), KITTI360_CALIB[1])
    if dataset == "NCLT":
        return nclt_calib()
    return np.eye(4)


HILTI_L2I = {"HILTI_2021": se3([0.999993918507834, 0.0012283821413574625, -0.0032596475280467258,
                                -0.00016947759535612024], [0.01001966915517371, -0.006645473484212856,
                                                           0.09473042428051345]),
             "HILTI_2022": se3([0.7071068, -0.7071068, 0.0, 0.0], [-0.001, -0.00855, 0.055])}


def kitti_line(M):
    return " ".join(repr(float(v)) for v in M[:3, :4].reshape(-1))


def pose_matrix(p):
    """a pose_dtype() record → 4 x 4 (normalised quaternion)"""
    return se3(p["quat"], p["tr"])
