"""Dataset sequences in the reference's layout (src/ct_icp/dataset.cpp: ADatasetSequence, NCLTIterator, PLYDirectory,
LoadDataset, LoadPoses), with every frame decoded and filtered on the device.

A frame is a dict: "xyz" (N, 3) and "t" (N,) torch CUDA tensors (a cticp_device_scan for Odometry.register_device
through `device_scan(frame)`), "frame_id", and "begin_pose" / "end_pose" (abi.Pose, or None without ground truth)
interpolated on the ground truth at the frame's first and largest timestamps (NCLT) or its minimum and maximum (PLY).
Options arrive as keyword arguments (load_dataset) or as a config.DatasetOptions read from a reference configuration
(load_dataset_from_options, which also builds SYNTHETIC sequences from scene YAML files).
"""
import os

import numpy as np

from . import _abi as abi

KITTI_SEQUENCES = ["%02d" % i for i in range(22)]
KITTI_360_SEQUENCES = ["00", "02", "03", "04", "05", "06", "07", "09", "10"]
KITTI_CARLA_SEQUENCES = ["Town0%d" % i for i in range(1, 8)]
HILTI_SEQUENCES = ["%02d" % i for i in range(12)]
# the sequence sizes of dataset.cpp (KITTI_SEQUENCES_SIZE, KITTI_360_SEQUENCES_SIZE, HILTI_SEQUENCES_SIZE; 5000 for
# KITTI_CARLA): a PLY directory has that many frames, and a missing file is an error when its frame is read
KITTI_SEQUENCES_SIZE = [4540, 1100, 4660, 800, 270, 2760, 1100, 1100, 4070, 1590, 1200, 920, 1060, 3280, 630, 1900,
                        1730, 490, 1800, 4980, 830, 2720]
KITTI_360_SEQUENCES_SIZE = [11500, 19230, 1029, 11399, 6722, 9697, 3160, 13954, 3742]
HILTI_SEQUENCES_SIZE = [895, 2004, 2641, 5824, 1130, 3308, 3503, 1357, 1995, 3992, 4298, 3749]
KITTI_CARLA_SEQUENCE_SIZE = 5000
NCLT_SEQUENCES = ["2012-01-08", "2012-01-15", "2012-01-22", "2012-02-02", "2012-02-04", "2012-02-05", "2012-02-12",
                  "2012-02-18", "2012-02-19", "2012-03-17", "2012-03-25", "2012-03-31", "2012-04-29", "2012-05-11",
                  "2012-05-26", "2012-06-15", "2012-08-04", "2012-08-20", "2012-09-28", "2012-10-28", "2012-11-04",
                  "2012-11-16", "2012-11-17", "2012-12-01", "2013-01-10", "2013-02-23", "2013-04-05"]


def device_scan(frame):
    """the abi.DeviceScan of a frame's xyz / t tensors"""
    xyz, t = frame["xyz"], frame["t"]
    codes = {"torch.float32": abi.DTYPE["float32"], "torch.float64": abi.DTYPE["float64"]}
    return abi.DeviceScan(xyz.data_ptr(), xyz.stride(0) * xyz.element_size(), t.data_ptr(),
                          t.stride(0) * t.element_size(), xyz.shape[0], codes[str(xyz.dtype)], codes[str(t.dtype)])


def pose_list(poses):
    """abi.Pose items of an array of abi.pose_dtype() (ground truth as Binding.ground_truth returns it), for
    Binding.continuous_trajectory"""
    import ctypes
    arr = np.ascontiguousarray(poses)
    out = []
    for i in range(len(arr)):
        p = abi.Pose()
        ctypes.memmove(ctypes.addressof(p), arr.ctypes.data + i * arr.itemsize, ctypes.sizeof(abi.Pose))
        out.append(p)
    return out


class _Sequence:
    """ADatasetSequence: HasNext / NextFrame / SkipFrame / SetInitFrame / SetMaxNumFrames / NumFrames / GroundTruth"""

    def __init__(self, binding, ground_truth=None, device=0):
        self.b = binding
        self.device = device
        self.gt = ground_truth                 # an array of abi.pose_dtype(), or None
        self._traj = None
        self.current = 0
        self.init = 0
        self.max_frames = -1

    def SetInitFrame(self, frame_index):
        self.init = self.current = frame_index

    def SetMaxNumFrames(self, n):
        self.max_frames = n

    def NumFrames(self):
        """AFileSequence::NumFrames: min(size - init, max_num_frames), or size - init without a maximum"""
        n = max(self._count() - self.init, 0)
        return n if self.max_frames < 0 else min(n, self.max_frames)

    def HasNext(self):
        """current < size, and current - init < max_num_frames when there is a maximum (dataset.cpp:421, :839-842)"""
        return self.current < self._count() and (self.max_frames < 0 or self.current - self.init < self.max_frames)

    def SkipFrame(self):
        if not self.HasNext():
            raise IndexError("no more frames in the sequence")
        self.current += 1

    def GroundTruth(self):
        return self.gt

    def close(self):
        """releases the device memory the reader holds between frames (a later NextFrame reopens it)"""
        self._traj = None

    def _poses(self, t_begin, t_end):
        if self.gt is None or len(self.gt) == 0:
            return None, None
        if self._traj is None:
            self._traj = self.b.continuous_trajectory(pose_list(self.gt), device=self.device)
        p = self._traj.interpolate(np.array([t_begin, t_end], dtype=np.float64))
        return p[0], p[1]

    def NextFrame(self):
        if not self.HasNext():
            raise IndexError("no more frames in the sequence")
        frame = self._read(self.current)
        frame["frame_id"] = self.current
        self.current += 1
        return frame


class NCLTSequence(_Sequence):
    """<root>/<seq>_vel/<seq>/velodyne_hits.bin read in whole-frame chunks of about chunk_bytes and decoded on the
    device, num_aggregated packets per frame; timestamps in microseconds, as the reference keeps them."""

    def __init__(self, binding, path, ground_truth=None, num_aggregated=220, chunk_bytes=64 << 20, device=0):
        super().__init__(binding, ground_truth, device)
        self.path, self.A, self.chunk = path, num_aggregated, chunk_bytes
        self._index()

    def _index(self):
        """every chunk's byte range and frame count: each chunk is opened once here, so a frame's bytes are known"""
        size = os.path.getsize(self.path)
        self.chunks, pos, first = [], 0, 0
        with open(self.path, "rb") as f:
            while pos < size:
                want = self.chunk
                while True:
                    f.seek(pos)
                    data = f.read(want)
                    final = pos + len(data) >= size
                    h = self.b.nclt_hits(data, self.A, final=final, device=self.device)
                    if h.num_frames or final:
                        break
                    want *= 2
                used = h.bytes_used if not final else len(data)
                self.chunks.append((pos, used, first, h.num_frames, final))
                first += h.num_frames
                pos += used
                h.close()
                if final:
                    break
        self._open = None

    def _count(self):
        return sum(c[3] for c in self.chunks)

    def close(self):
        if self._open is not None:
            self._open[1].close()
            self._open = None
        super().close()

    def _read(self, k):
        for (pos, used, first, nf, final) in self.chunks:
            if first <= k < first + nf:
                break
        if self._open is None or self._open[0] != pos:
            with open(self.path, "rb") as f:
                f.seek(pos)
                data = f.read(used)
            self._open = (pos, self.b.nclt_hits(data, self.A, final=final, device=self.device))
        h = self._open[1]
        out = h.read(first=k - first, m=1)
        info = h.frame_info(k - first, 1)[0]
        begin, end = self._poses(info["t_first"], info["t_max"]) if info["num_points"] else (None, None)
        return {"xyz": out["xyz"], "t": out["t"], "begin_pose": begin, "end_pose": end}


class PLYDirectory(_Sequence):
    """`size` files frame_%04d.ply (KITTI) or frame_%05d.ply (KITTI-360, HILTI) of a directory, decoded on the host,
    copied to the device and filtered there with kitti_frame_filter when `kitti_filter` (KITTI, KITTI_raw, KITTI_360).
    The size comes from the dataset's table, as in the reference; a missing file raises when its frame is read."""

    def __init__(self, binding, directory, size, digits=4, kitti_filter=False, ground_truth=None, device=0):
        super().__init__(binding, ground_truth, device)
        self.dir, self.digits, self.filter = directory, digits, kitti_filter
        self.n = size

    def _name(self, k):
        return os.path.join(self.dir, ("frame_%0" + str(self.digits) + "d.ply") % k)

    def _count(self):
        return self.n

    def _read(self, k):
        import torch
        with open(self._name(k), "rb") as f:
            data = f.read()
        _, rec = self.b.ply_records(data)
        dev = torch.device("cuda", self.device)
        xyz = torch.from_numpy(np.stack([rec["x"], rec["y"], rec["z"]], 1).astype(rec["x"].dtype)).to(dev)
        if self.filter:
            xyz = self.b.kitti_frame_filter(xyz, device=self.device, in_place=True)
        has_t = "t" in rec.dtype.names
        t = torch.from_numpy(rec["t"].astype(np.float64) if has_t else np.zeros(len(rec))).to(dev)
        begin = end = None
        if has_t and len(rec):
            mm = self.b.scan_time_ranges(t, torch.tensor([len(rec)], dtype=torch.int64), device=self.device)
            begin, end = self._poses(*mm[0].tolist())
        return {"xyz": xyz, "t": t, "begin_pose": begin, "end_pose": end}


def write_ply_frames(binding, xyz, t, frame_ends, directory, digits=4, first_index=0, device=0):
    """Frames of a scan sequence as frame_%0<digits>d.ply files in `directory` (numbered from first_index) in the
    layout of the reference's WPoint3D::FloatSchemaMapper (io.cxx:842-855): element vertex, float x y z timestamp. xyz
    (N, 3) and t (N,) are CUDA tensors or NumPy arrays of any float or integer type, frame_ends the frames' ends. All
    frames are encoded in one device call and copied to the host once; PLYDirectory reads the directory back. Returns
    the paths."""
    cols = [("vertex", k, "float", xyz[:, i]) for i, k in enumerate("xyz")] + [("vertex", "timestamp", "float", t)]
    if not any(hasattr(c[3], "is_cuda") and c[3].is_cuda for c in cols):
        import torch
        dev = torch.device("cuda", device)
        cols = [(e, k, p, torch.as_tensor(np.asarray(a)).to(dev)) for e, k, p, a in cols]
    data, offsets = binding.ply_write(cols, file_ends=frame_ends, device=device)
    data, offsets = data.cpu().numpy(), offsets.cpu().numpy()
    os.makedirs(directory, exist_ok=True)
    paths = []
    for k in range(len(offsets) - 1):
        path = os.path.join(directory, ("frame_%0" + str(digits) + "d.ply") % (first_index + k))
        with open(path, "wb") as f:
            f.write(data[offsets[k]:offsets[k + 1]].tobytes())
        paths.append(path)
    return paths

def _read_gt(binding, dataset, path, sequence_id):
    if not os.path.exists(path):
        return None
    with open(path, "rb") as f:
        return binding.ground_truth(dataset, f.read(), sequence_id)


def load_dataset(binding, dataset, root, sequences=None, device=0, **options):
    """LoadDataset: the sequences of `dataset` found under `root` by the reference's directory names (all of them, or
    those named in `sequences`), each with its ground truth when the file the reference reads is present. Returns a
    list of (name, sequence)."""
    out = []
    if dataset == "NCLT":
        for i, name in enumerate(NCLT_SEQUENCES):
            if sequences is not None and name not in sequences:
                continue
            hits = os.path.join(root, name + "_vel", name, "velodyne_hits.bin")
            if not os.path.exists(hits):
                continue
            gt = _read_gt(binding, "NCLT", os.path.join(root, name + "_vel", name, "groundtruth_%s.csv" % name), i)
            out.append((name, NCLTSequence(binding, hits, gt, device=device, **options)))
        return out
    names = {"KITTI": KITTI_SEQUENCES, "KITTI_raw": KITTI_SEQUENCES, "KITTI_360": KITTI_360_SEQUENCES,
             "KITTI_CARLA": KITTI_CARLA_SEQUENCES, "HILTI_2021": HILTI_SEQUENCES, "HILTI_2022": HILTI_SEQUENCES}
    sizes = {"KITTI": KITTI_SEQUENCES_SIZE, "KITTI_raw": KITTI_SEQUENCES_SIZE, "KITTI_360": KITTI_360_SEQUENCES_SIZE,
             "KITTI_CARLA": [KITTI_CARLA_SEQUENCE_SIZE] * 7, "HILTI_2021": HILTI_SEQUENCES_SIZE,
             "HILTI_2022": HILTI_SEQUENCES_SIZE}
    if dataset not in names:
        raise ValueError("unknown dataset %r" % dataset)
    for i, name in enumerate(names[dataset]):
        if sequences is not None and name not in sequences:
            continue
        seq_dir = os.path.join(root, name)
        frames = os.path.join(seq_dir, "frames")
        if not os.path.isdir(frames):
            continue
        gt = None
        if dataset in ("KITTI", "KITTI_raw", "KITTI_360"):
            gt = _read_gt(binding, dataset, os.path.join(seq_dir, name + ".txt"), i)
        elif dataset == "KITTI_CARLA":
            gt = _read_gt(binding, dataset, os.path.join(seq_dir, "poses_gt.txt"), i)
        digits = 4 if dataset in ("KITTI", "KITTI_raw", "KITTI_CARLA") else 5
        out.append((name, PLYDirectory(binding, frames, sizes[dataset][i], digits,
                                       dataset in ("KITTI", "KITTI_raw", "KITTI_360"), gt, device)))
    return out


class SyntheticSequence(_Sequence):
    """SyntheticSequence (dataset.cpp:693-790) of a scene, the dict config.yaml_to_synthetic_scene reads: frame k spans
    ground-truth poses k and k + 1, sampled at sample_frequency along the scene's trajectory, and its points are
    generated on the device (Binding.synthetic_sequence, with `seed`) when the first frame is read. The ground truth
    is the sampled poses relative to the first. As the reference's HasNext, max_num_frames does not shorten it."""

    def __init__(self, binding, spec, seed=0, device=0):
        super().__init__(binding, None, device)
        self.spec, self.seed = spec, seed
        self._data = None
        self.gt = binding.synthetic_sequence(spec, seed=seed, num_frames=0, device_index=device)["ground_truth"]

    def _count(self):
        return max(len(self.gt) - 1, 0)

    def NumFrames(self):
        return len(self.gt)        # seq_info.sequence_size: the number of ground-truth poses

    def HasNext(self):
        return self.current < self._count()

    def _read(self, k):
        if self._data is None:
            d = self.b.synthetic_sequence(self.spec, seed=self.seed, device=True, device_index=self.device)
            self._data = (d["xyz"], d["t"], [0] + d["frame_ends"].tolist())
        xyz, t, ends = self._data
        begin, end = pose_list(self.gt[k:k + 2])
        return {"xyz": xyz[ends[k]:ends[k + 1]], "t": t[ends[k]:ends[k + 1]], "begin_pose": begin, "end_pose": end}

    def close(self):
        self._data = None
        super().close()


def load_dataset_from_options(binding, options, device=0):
    """Dataset::LoadDataset (dataset.cpp:1214-1260) of a config.DatasetOptions: the dataset's sequences found under
    root_path, each labelled <DATASET>_<name> (e.g. KITTI_raw_00, NCLT_2012-01-08, SYNTHETIC_courtyard). With
    use_all_datasets false only the sequences of sequence_options are kept, each with its start_frame_id and
    max_num_frames, and a named sequence that is not found is an error. SYNTHETIC: every <root_path>/*.yaml is one
    sequence, named by the file's stem. Sequences come in name order (the reference's order is the directory
    iterator's). Returns a list of (label, sequence)."""
    from . import config
    if options.dataset is None or options.dataset == "PLY_DIRECTORY":
        raise config.ConfigError("The dataset %s cannot be defined from the config" % (options.dataset,))
    if not os.path.exists(options.root_path):
        raise config.ConfigError("The path to the root directory does not exist: %s" % options.root_path)
    wanted = None if options.use_all_datasets else {s.sequence_name: s for s in options.sequence_options}
    if options.dataset == "SYNTHETIC":
        found = []
        for fname in sorted(os.listdir(options.root_path)):
            path = os.path.join(options.root_path, fname)
            stem, ext = os.path.splitext(fname)
            if not os.path.isfile(path) or ext != ".yaml" or (wanted is not None and stem not in wanted):
                continue
            spec = config.yaml_to_synthetic_scene(config.load_config(path))
            found.append((stem, SyntheticSequence(binding, spec, device=device)))
    else:
        kw = {"num_aggregated": options.nclt_num_aggregated_pc} if options.dataset == "NCLT" else {}
        found = load_dataset(binding, options.dataset, options.root_path,
                             None if wanted is None else list(wanted), device=device, **kw)
        found.sort(key=lambda x: x[0])
    if wanted is not None:
        if len(found) != len(wanted):
            raise config.ConfigError("Could not find all the sequences in `sequence_options`")
        for name, seq in found:
            seq.SetInitFrame(wanted[name].start_frame_id)
            seq.SetMaxNumFrames(wanted[name].max_num_frames)
    return [(options.dataset + "_" + name, seq) for name, seq in found]
