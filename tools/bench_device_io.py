"""Per-frame time of RegisterFrame from host buffers, from a staged scan (RegisterStaged) and from CUDA tensors
(cticp_odometry_register_device), and of the summary's point vectors copied back (get_points) against written to device
memory (points_device), on the bench workload (BASELINE.json configs[1], bench.py's options and scans).

Each mode has its own odometry over the same frames; the three modes take turns frame by frame, in an order that rotates
every round. A step is host-timed: the queue is drained first, the clock stops when the frame's map-update tail has
completed (last_timing), as in bench.py's end-to-end pass. Egress is timed after that, on the host-buffer odometry
(points_into the three vectors as 64-byte records) and on the tensor odometry (points_device of the three vectors, world
coordinates + timestamps, float64, then a device synchronise). The card name and power limit come from a read-only
nvidia-smi query in the same run.

usage: python tools/bench_device_io.py [--steps 40] [--warmup 5] [--preroll 20] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
import ct_icp_b200  # noqa: E402
from ct_icp_b200 import _abi as abi  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def stats(ms):
    a = np.asarray(ms)
    return {"mean_ms": float(a.mean()), "median_ms": float(np.median(a)), "min_ms": float(a.min()),
            "max_ms": float(a.max()), "n": int(len(a))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--preroll", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    eng = ct_icp_b200.engine()
    first = args.preroll + args.warmup
    seq = bench.make_scans(first + args.steps, bench.WORKLOADS["kitti64_gn"][0])
    mods = ["host", "staged", "device"]
    ods = {m: eng.odometry(bench.make_options(eng)) for m in mods}
    slots = [ods["staged"].stage_frame(s["xyz"], s["t"]) for s in seq]
    dev = [(torch.from_numpy(s["xyz"]).cuda(), torch.from_numpy(s["t"]).cuda()) for s in seq]
    cap = max(len(s["xyz"]) for s in seq)
    bufs = [np.zeros(cap, dtype=abi.wpoint_dtype()) for _ in range(3)]
    torch.cuda.synchronize()

    def register(mode, i):
        s = seq[i]
        if mode == "host":
            return ods[mode].RegisterFrame(s["xyz"], s["t"], s["frame_idx"])
        if mode == "staged":
            return ods[mode].RegisterStaged(slots[i], s["frame_idx"])
        return ods[mode].RegisterFrame(dev[i][0], dev[i][1], s["frame_idx"])

    times = {m: [] for m in mods}
    egress = {"get_points": [], "points_device": []}
    poses = {m: [] for m in mods}
    for i in range(first + args.steps):
        timed = i >= first
        order = mods[i % 3:] + mods[:i % 3]
        for m in order:
            torch.cuda.synchronize()
            ods[m].last_timing()
            t0 = time.perf_counter()
            sm = register(m, i)
            ods[m].last_timing()
            dt = (time.perf_counter() - t0) * 1e3
            assert sm.success, (m, i, sm.error_message)
            poses[m].append(bench.pose_vector(sm))
            if timed:
                times[m].append(dt)
            if m == "host":
                t0 = time.perf_counter()
                for w in (1, 2, 0):
                    ods[m].points_into(w, bufs[w])
                if timed:
                    egress["get_points"].append((time.perf_counter() - t0) * 1e3)
            elif m == "device":
                t0 = time.perf_counter()
                for w in (1, 2, 0):
                    ods[m].points_device(w, world=True, with_timestamps=True)
                torch.cuda.synchronize()
                if timed:
                    egress["points_device"].append((time.perf_counter() - t0) * 1e3)
    same = all(np.array_equal(np.array(poses["host"]), np.array(poses[m])) for m in mods)
    out = {"card": card(), "workload": bench.WORKLOAD, "steps": args.steps, "warmup": args.warmup,
           "preroll": args.preroll, "points_per_scan": float(np.mean([len(s["xyz"]) for s in seq[first:]])),
           "register_ms": {m: stats(times[m]) for m in mods}, "egress_ms": {k: stats(v) for k, v in egress.items()},
           "poses_identical_across_modes": bool(same)}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_device_io.json"), "w") as f:
            f.write(line + "\n")
    for od in ods.values():
        od.close()


if __name__ == "__main__":
    main()
