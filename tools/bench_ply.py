#!/usr/bin/env python
"""Throughput of the PLY writer on the device (include/cticp.h, "PLY files").

Workloads:
  (a) a 20M-point world-cloud-size export from fp64 columns (x, y, z, t of an (N, 4) array): float xyz + double
      timestamp (20-byte records) and double xyz (24-byte records);
  (b) 100 HDL-64 sweeps of the suburb scene (synthetic.UrbanScene(1234)) as frame_%04d.ply files in the reference's
      FloatSchemaMapper layout (float x y z timestamp): one call for all files against 100 calls of one file;
  (c) for context, a NumPy structured-array writer on the host for (a)'s first layout, from host arrays.
Times are medians of --reps CUDA-event windows around cticp_ply_write_device into a preallocated buffer (no host
synchronisation inside the window). The algorithmic bytes are the column bytes read plus the file bytes written; the
share is their rate over 3.35 TB/s (the H100 SXM data sheet's HBM3 bandwidth). Prints one JSON line with the card's
name and power limit.
usage: python tools/bench_ply.py [--reps 20] [--points 20000000]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import ct_icp_b200  # noqa: E402
from ct_icp_b200 import _abi as abi  # noqa: E402
from ct_icp_b200 import synthetic as syn  # noqa: E402
import lidar_sim_ref as lref  # noqa: E402

PEAK = 3.35e12


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


class Call:
    """one prepared cticp_ply_write_device call: columns (element, name, ply code, 1-D tensor), file ends (tensor)"""

    def __init__(self, eng, cols, ends, n):
        self.fn = eng.fn("ply_write_device")
        self.keep = [(e.encode(), k.encode()) for e, k, _, _ in cols]
        self.props = (abi.PlyProperty * len(cols))(*[
            abi.PlyProperty(ek[0], ek[1], p, abi.PLY_SRC_DTYPE[str(a.dtype).replace("torch.", "")], a.data_ptr(),
                            a.stride(0) * a.element_size()) for (e, k, p, a), ek in zip(cols, self.keep)])
        self.n, self.ends, self.m = n, ends, ends.numel()
        self.offsets = torch.empty(self.m + 1, dtype=torch.int64, device="cuda")
        self.stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        self.go(None, 0)
        self.total = int(self.offsets[-1].item())
        self.out = torch.empty(self.total, dtype=torch.uint8, device="cuda")
        self.read = sum(a.element_size() * n for _, _, _, a in cols)

    def go(self, out=0, cap=None):
        rc = self.fn(0, self.props, len(self.props), self.n, self.ends.data_ptr(), self.m,
                     self.out.data_ptr() if out == 0 else out, self.total if cap is None else cap,
                     self.offsets.data_ptr(), self.stream)
        assert rc == 0, rc


def rate(ms, nbytes):
    return {"ms": round(ms, 4), "bytes": int(nbytes), "GB_per_s": round(nbytes / ms / 1e6, 1),
            "share_of_3_35_TBps": round(nbytes / ms / 1e-3 / PEAK, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--points", type=int, default=20_000_000)
    args = ap.parse_args()
    eng = ct_icp_b200.engine()
    res = {"card": card()}
    n = args.points
    g = torch.Generator(device="cuda").manual_seed(1)
    xyzt = torch.rand((n, 4), dtype=torch.float64, device="cuda", generator=g)
    end = torch.tensor([n], dtype=torch.int64, device="cuda")
    F, D = abi.DTYPE["float32"], abi.DTYPE["float64"]
    layouts = {"float_xyz_double_t_20B": [("vertex", k, F, xyzt[:, i]) for i, k in enumerate("xyz")] +
               [("vertex", "timestamp", D, xyzt[:, 3])],
               "double_xyz_24B": [("vertex", k, D, xyzt[:, i]) for i, k in enumerate("xyz")]}
    for name, cols in layouts.items():
        c = Call(eng, cols, end, n)
        res["a_" + name] = rate(timed(c.go, args.reps), c.read + c.total)
        del c
    # (b) 100 HDL-64 sweeps
    scene, traj = syn.UrbanScene(1234, profile="suburb"), syn.Trajectory(height=1.73)
    sc = eng.lidar_scene(scene.boxes, scene.cyl)
    tr = eng.continuous_trajectory(lref.trajectory_poses(traj, 100 * syn.HDL64.period + 0.2))
    sw = sc.sweeps(tr, syn.HDL64, [(k * syn.HDL64.period, k) for k in range(100)], seed=2)
    xyz, t = sw["xyz"], sw["t"]
    ends = sw["frame_ends"].to(torch.int64)
    cols = [("vertex", k, F, xyz[:, i]) for i, k in enumerate("xyz")] + [("vertex", "timestamp", F, t)]
    batch = Call(eng, cols, ends, xyz.shape[0])
    res["b_points"] = int(xyz.shape[0])
    res["b_one_call_100_files"] = rate(timed(batch.go, args.reps), batch.read + batch.total)
    e = [0] + ends.cpu().tolist()
    singles = [Call(eng, [(el, k, p, a[e[i]:e[i + 1]]) for el, k, p, a in cols],
                    torch.tensor([e[i + 1] - e[i]], dtype=torch.int64, device="cuda"), e[i + 1] - e[i])
               for i in range(100)]

    def all_singles():
        for s in singles:
            s.go()
    res["b_100_calls_of_one_file"] = rate(timed(all_singles, args.reps), batch.read + batch.total)
    ok = batch.out.cpu().numpy().tobytes() == b"".join(s.out.cpu().numpy().tobytes() for s in singles)
    res["b_files_equal"] = ok
    # (c) NumPy on the host, for context
    h = xyzt.cpu().numpy()
    head = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\n"
            "property float z\nproperty double timestamp\nend_header\n" % n).encode()
    t0 = time.perf_counter()
    rec = np.empty(n, dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("t", "<f8")])
    rec["x"], rec["y"], rec["z"], rec["t"] = h[:, 0], h[:, 1], h[:, 2], h[:, 3]
    data = head + rec.tobytes()
    ms = (time.perf_counter() - t0) * 1e3
    res["c_numpy_host_20B_ms"] = round(ms, 2)
    c = Call(eng, layouts["float_xyz_double_t_20B"], end, n)
    c.go()
    res["c_equals_device_file"] = c.out.cpu().numpy().tobytes() == data
    print(json.dumps(res))


if __name__ == "__main__":
    main()
