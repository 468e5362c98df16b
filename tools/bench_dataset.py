#!/usr/bin/env python
"""Throughput of the dataset readers on the device (include/cticp.h, "Dataset sequences").

Workloads, on NCLT-shape streams packed from HDL-32 sweeps of the suburb scene (synthetic.UrbanScene(1234)), 220
packets per frame, hits quantised to 5 mm:
  * the decode of one frame and of 100 frames per call into a device sink (x, y, z, t fp64): microseconds per call
    (CUDA events, median of --reps after a warm-up) and GB/s of hit bytes read;
  * the index of a 100-frame stream (cticp_nclt_open on host bytes: copy, magic scan, chain check, host frames);
  * the KITTI filter on a 120k-point float32 frame, in place;
  * bytes over PCIe per frame: the raw packets against x, y, z, t in fp64;
  * file bytes to a registered frame: open on one frame's host bytes, decode into device memory, register_device.
Prints one JSON line with the card's name and power limit.
usage: python tools/bench_dataset.py [--reps 20]"""
import argparse
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
import dataset_ref as ref  # noqa: E402
import lidar_sim_ref as lref  # noqa: E402
from test_gpu_parity import _sequence_options  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def timed(fn, reps):
    """median milliseconds of fn() on torch's current stream"""
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


def nclt_stream(eng, frames, A=220):
    scene, traj = syn.UrbanScene(1234, profile="suburb"), syn.Trajectory(height=1.0)
    sc = eng.lidar_scene(scene.boxes, scene.cyl)
    tr = eng.continuous_trajectory(lref.trajectory_poses(traj, frames * 0.1 + 0.2))
    out = sc.sweeps(tr, syn.HDL32, [(k * syn.HDL32.period, k) for k in range(frames)], seed=1, device=False)
    ends = out["frame_ends"].astype(np.int64)
    q = ref.quantise(out["xyz"])
    chunks, a = [], 0
    for b in ends:
        bounds = np.linspace(a, b, A + 1).astype(np.int64)
        for k in range(A):
            ut = 1_300_000_000_000_000 + int(round(out["t"][min(bounds[k], len(q) - 1)] * 1e6))
            chunks.append(ref.pack_packet(ut, q[bounds[k]:bounds[k + 1]]))
        a = b
    return b"".join(chunks), chunks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    eng = ct_icp_b200.engine()
    stream = lambda: torch.cuda.current_stream().cuda_stream  # noqa: E731
    res = {"card": card()}
    data, chunks = nclt_stream(eng, 100)
    h = eng.nclt_hits(data, 220)
    hits = h.num_hits
    rec = torch.empty((hits, 32), dtype=torch.uint8, device="cuda")
    ends = torch.empty(100, dtype=torch.int64, device="cuda")
    sink = abi.CloudSink(rec.data_ptr(), hits, 32, 0, abi.DTYPE["float64"], 24, abi.DTYPE["float64"], 0)
    info = h.frame_info()
    for m in (1, 100):
        ms = timed(lambda: h.read_device(0, m, sink, ends.data_ptr(), stream()), args.reps)
        n = int(info["num_points"][:m].sum())
        res["decode_%d_frames" % m] = {"us_per_call": round(ms * 1e3, 2), "us_per_frame": round(ms * 1e3 / m, 2),
                                        "points": n, "hit_GBps": round(8 * n / (ms * 1e-3) / 1e9, 1)}
    t0 = time.perf_counter()
    for _ in range(3):
        eng.nclt_hits(data, 220).close()
    res["open_100_frames_ms"] = round((time.perf_counter() - t0) / 3 * 1e3, 2)
    res["stream_MB"] = round(len(data) / 1e6, 2)
    pts = int(info["num_points"].mean())
    raw = len(data) / 100
    res["pcie_bytes_per_frame"] = {"points": pts, "raw_packets": int(raw), "decoded_xyzt_fp64": 32 * pts,
                                   "ratio": round(32 * pts / raw, 2)}
    # the KITTI filter, in place on 120k float32 records of 16 bytes (x y z t)
    rng = np.random.default_rng(0)
    x = torch.from_numpy(rng.uniform(-60, 60, (120_000, 4)).astype(np.float32)).cuda()
    scan = abi.DeviceScan(x.data_ptr(), 16, None, 0, len(x), abi.DTYPE["float32"], 0)
    fs = abi.CloudSink(x.data_ptr(), len(x), 16, 0, abi.DTYPE["float32"], 0, 0, 0)
    ms = timed(lambda: eng.check(eng.fn("kitti_frame_filter_device")(0, scan, fs, stream())), args.reps)
    res["kitti_filter_120k_us"] = round(ms * 1e3, 2)
    # file bytes to a registered frame
    od = eng.odometry(_sequence_options(eng, "GN", init_num_frames=3))
    per = []
    for k in range(12):
        frame = b"".join(chunks[k * 220:(k + 1) * 220])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        hk = eng.nclt_hits(frame, 220)
        d = hk.read()
        n = d["xyz"].shape[0]
        s = abi.DeviceScan(d["xyz"].data_ptr(), 32, d["t"].data_ptr(), 32, n, abi.DTYPE["float64"],
                           abi.DTYPE["float64"])
        sm = od.register_device(s, k, stream=stream())
        per.append((time.perf_counter() - t0) * 1e3)
        assert sm.success, sm.error_message
    res["bytes_to_registered_frame_ms"] = {"median": round(float(np.median(per[3:])), 3),
                                           "min": round(float(np.min(per[3:])), 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
