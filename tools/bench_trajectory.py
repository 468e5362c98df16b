"""Throughput of RawPointsToWorldPoints along a continuous trajectory (cticp_trajectory_transform[_device]).

64 concatenated bench-size scans (130,000 points each, ~8.3M points; float32 x, y, z, pad as an (N, 4) tensor and float64
timestamps) along an odometry-shaped trajectory of 64 frames (begin and end pose each), written as float64 world x, y, z:
  - device path, both lookup modes (by timestamp; by frame id with one segment per scan): CUDA events around the call
    on its stream, points/s, and the bytes the kernel must move (20 B read + 24 B written per point) per second as a
    share of the data-sheet HBM bandwidth of the card;
  - host path (host records in, host sink out, the copies included): wall clock around the call;
  - the CPU restatement of the reference (one point at a time, fp64 + libm) on a 200,000-point slice: wall clock.
Prints the GPU's name and power limit with the numbers, and one JSON line last. Writes nothing to the tree; the JSON goes
to --out when given.

    python tools/bench_trajectory.py [--reps 20] [--out /tmp/bench_trajectory.json]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

SCANS, PER_SCAN = 64, 130000
HBM_BYTES_PER_S = {"H100 80GB HBM3": 3.35e12, "H100 PCIe": 2.0e12}   # NVIDIA data sheets (SXM5 / PCIe)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, sm = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": sm}
    except Exception as e:   # the numbers are still printed; the card is then named by torch alone
        return {"name": None, "power_limit": "unknown (%s)" % e, "max_sm_clock": None}


def trajectory_poses(abi, rng):
    poses = []
    q, tr, t = np.array([0.0, 0.0, 0.0, 1.0]), np.zeros(3), 1000.0
    for k in range(SCANS):
        for e in range(2):
            q = q + rng.normal(scale=0.01, size=4)
            q /= np.linalg.norm(q)
            tr = tr + rng.normal(scale=0.5, size=3)
            p = abi.Pose.make(quat=q, tr=tr, dest_timestamp=t + 0.1 * e, dest_frame_id=k)
            poses.append(p)
        t += 0.1
    return poses


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--oracle-points", type=int, default=200000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_trajectory: no CUDA device (this benchmark measures the GPU path only)")
    import ct_icp_b200
    from ct_icp_b200 import _abi as abi
    from oracle_trajectory_lib import trajectory_oracle

    info = gpu_info()
    info["torch_name"] = torch.cuda.get_device_name(0)
    peak = next((v for k, v in HBM_BYTES_PER_S.items() if k in (info["name"] or info["torch_name"])), 3.35e12)
    rng = np.random.default_rng(2026)
    poses = trajectory_poses(abi, rng)
    eng = ct_icp_b200.engine()
    te = eng.continuous_trajectory(poses)
    n = SCANS * PER_SCAN
    g = torch.Generator(device="cuda").manual_seed(1)
    xyz = (torch.rand((n, 4), generator=g, device="cuda", dtype=torch.float32) - 0.5) * 200.0
    fr = torch.arange(n, device="cuda") // PER_SCAN
    P = te.poses()
    b = torch.from_numpy(P["dest_timestamp"][0::2].copy()).cuda()
    t = b[fr] + torch.rand(n, generator=g, device="cuda", dtype=torch.float64) * 0.1
    out = torch.empty((n, 3), dtype=torch.float64, device="cuda")
    scan = abi.DeviceScan(xyz.data_ptr(), 16, t.data_ptr(), 8, n, abi.DTYPE["float32"], abi.DTYPE["float64"])
    sink = abi.CloudSink(out.data_ptr(), n, 24, 0, abi.DTYPE["float64"], 0, 0, 1)
    segments = (np.arange(1, SCANS + 1, dtype=np.uint64) * PER_SCAN, np.arange(SCANS, dtype=np.uint32))
    bytes_per_point = 3 * 4 + 8 + 3 * 8   # x, y, z read, t read, world written (the pad column is skipped by the loads)
    stream = torch.cuda.current_stream()
    results = {"gpu": info, "points": n, "scans": SCANS, "bytes_per_point": bytes_per_point,
               "hbm_peak_bytes_per_s": peak}

    for mode, seg in (("timestamp", None), ("frame_id", segments)):
        for _ in range(args.warmup):
            te.transform_device(scan, sink, seg, stream.cuda_stream)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        ev[0].record(stream)
        for _ in range(args.reps):
            te.transform_device(scan, sink, seg, stream.cuda_stream)
        ev[1].record(stream)
        torch.cuda.synchronize()
        ms = ev[0].elapsed_time(ev[1]) / args.reps
        results["device_" + mode] = {"ms_per_call": ms, "points_per_s": n / (ms * 1e-3),
                                     "bytes_per_s": n * bytes_per_point / (ms * 1e-3),
                                     "share_of_hbm_peak": n * bytes_per_point / (ms * 1e-3) / peak}

    # host path: the same records in host memory, host sink; wall clock around the (synchronous) call
    xyz_h, t_h = xyz.cpu().numpy(), t.cpu().numpy()
    rec = np.zeros(n, dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("pad", "<f4"), ("t", "<f8")])
    rec["x"], rec["y"], rec["z"], rec["t"] = xyz_h[:, 0], xyz_h[:, 1], xyz_h[:, 2], t_h
    sink_h = np.zeros(n, dtype=[("x", "<f8"), ("y", "<f8"), ("z", "<f8")])
    te.transform_records(rec, sink_h, segments)
    reps_h = max(2, args.reps // 5)
    t0 = time.perf_counter()
    for _ in range(reps_h):
        te.transform_records(rec, sink_h, segments)
    s = (time.perf_counter() - t0) / reps_h
    results["host_frame_id"] = {"ms_per_call": s * 1e3, "points_per_s": n / s}
    te.transform_device(scan, sink, segments, stream.cuda_stream)
    torch.cuda.synchronize()
    results["host_equals_device"] = bool(out.cpu().numpy().tobytes() == sink_h.view(np.float64).tobytes())

    # the reference's loop on the CPU (one point at a time) on a slice
    m = min(args.oracle_points, n)
    to = trajectory_oracle().continuous_trajectory(poses)
    sink_o = np.zeros(m, dtype=sink_h.dtype)
    seg_m = (np.minimum(segments[0], m), segments[1])
    t0 = time.perf_counter()
    to.transform_records(rec[:m], sink_o, seg_m)
    s = time.perf_counter() - t0
    results["cpu_reference_loop"] = {"points": m, "ms": s * 1e3, "points_per_s": m / s}
    results["max_abs_diff_vs_cpu_m"] = float(np.abs(sink_o.view(np.float64) - sink_h[:m].view(np.float64)).max())

    print("GPU: %s, power limit %s, max SM clock %s" % (info["name"] or info["torch_name"], info["power_limit"],
                                                        info["max_sm_clock"]))
    for k in ("device_timestamp", "device_frame_id"):
        r = results[k]
        print("%-17s %8.3f ms  %7.2f Gpoint/s  %7.1f GB/s  %5.1f%% of %.2f TB/s" % (
            k, r["ms_per_call"], r["points_per_s"] / 1e9, r["bytes_per_s"] / 1e9, 100 * r["share_of_hbm_peak"], peak / 1e12))
    print("host_frame_id     %8.1f ms  %7.3f Gpoint/s (copies included)" % (results["host_frame_id"]["ms_per_call"],
                                                                            results["host_frame_id"]["points_per_s"] / 1e9))
    print("cpu reference     %8.1f ms for %d points: %.2f Mpoint/s" % (results["cpu_reference_loop"]["ms"], m,
                                                                       results["cpu_reference_loop"]["points_per_s"] / 1e6))
    line = json.dumps(results)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
