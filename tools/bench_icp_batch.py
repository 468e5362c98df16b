"""B solo cticp_icp_register calls against one batched call (cticp_icp_register_batch for solver GN,
cticp_icp_register_batch_ex for CERES and ROBUST), on one map.

The map is built from the HDL-64 synthetic sequence (frames 0..2 registered by the CPU oracle, as the GPU parity tests
do); the B problems are frame 3's keypoints (1.0 m grid, or its first --small keypoints) at B initial poses perturbed by
a few centimetres. Reported per (B, K):
  - host-timed end to end, per problem: median over --repeats of B solo calls / one batch call (each synchronising)
  - device time of the persistent launches (torch.profiler, separate run): k_gn_persistent for GN, k_lm_persistent for
    CERES / ROBUST; Σ over the B solo launches / the batch
The card name and power limit come from a read-only nvidia-smi query in the same run.

usage: python tools/bench_icp_batch.py [--solver GN|CERES|ROBUST] [--batches 1,2,4,8,16,32] [--small 500]
                                       [--repeats 20] [--warmup 3]
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

import ct_icp_b200  # noqa: E402
from ct_icp_b200 import _abi as abi  # noqa: E402
from ct_icp_b200 import synthetic as syn  # noqa: E402
from oracle_lib import oracle  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def registration_case():
    orc = oracle()
    seq = syn.make_sequence(4, syn.HDL64, seed=1234)
    o = orc.default_odometry_options()
    o.ct_icp_options.solver = abi.SOLVER["GN"]
    o.ct_icp_options.min_number_neighbors = 10
    o.map_options = orc.legacy_map_options(1.0, 20, 0.1)
    o.debug_print = 0
    od = orc.odometry(o)
    for s in seq[:3]:
        assert od.RegisterFrame(s["xyz"], s["t"], s["frame_idx"]).success
    map_xyz, _ = od.GetMapPointer().export(0)
    s = seq[3]
    idx = orc.grid_sample_indices(s["xyz"], 1.0)
    kp = np.zeros(len(idx), dtype=abi.wpoint_dtype())
    kp["raw"] = s["xyz"][idx]
    kp["timestamp"] = s["t"][idx]
    traj = od.Trajectory()
    frame = traj[-1].copy()
    frame.begin_pose = traj[-1].end_pose.copy()
    frame.begin_pose.dest_timestamp = float(s["t"].min())
    frame.end_pose.dest_timestamp = float(s["t"].max())
    return map_xyz, kp, frame, traj[-1]


def perturbed(frame, k):
    f = frame.copy()
    d = 0.03 * np.array([np.cos(1.3 * k), np.sin(0.7 * k), 0.3 * np.cos(2.1 * k)])
    f.begin_pose.tr = tuple(np.array(f.begin_pose.tr) + d)
    f.end_pose.tr = tuple(np.array(f.end_pose.tr) + d)
    return f


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,2,4,8,16,32")
    ap.add_argument("--small", type=int, default=500, help="keypoints of the small problems (a truncated set)")
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--solver", default="GN", choices=sorted(abi.SOLVER))
    args = ap.parse_args()
    batches = [int(b) for b in args.batches.split(",")]

    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.init()
    eng = ct_icp_b200.engine()
    map_xyz, kp_full, frame, prev = registration_case()
    mopt = eng.legacy_map_options(1.0, 20, 0.1)
    mopt.capacity_voxels = 1 << 18
    m = eng.voxel_map(mopt)
    m.insert(map_xyz)
    io = eng.default_icp_options()
    io.solver = abi.SOLVER[args.solver]
    io.min_number_neighbors = 10
    io.num_iters_icp = 8
    if args.solver == "CERES":   # the reference's default options otherwise: nearest-neighbor strategy
        io.loss_function = abi.LOSS["CAUCHY"]
        io.num_iters_icp = 4
    elif args.solver == "ROBUST":
        io.num_iters_icp = 4
        io.max_num_residuals = 1000
        io.weight_alpha, io.weight_neighborhood = 0.9, 0.1
        io.min_number_neighbors, io.max_number_neighbors = 8, 20
        io.loss_function = abi.LOSS["CAUCHY"]
        io.ls_max_num_iters, io.ls_sigma = 8, 0.1
        io.max_dist_to_plane_ct_icp, io.outlier_distance = 0.5, 0.8
        io.threshold_linearity, io.threshold_planarity = 0.9, 0.8
    kernel = "k_gn_persistent" if args.solver == "GN" else "k_lm_persistent"
    mm = eng.default_odometry_options().default_motion_model
    info = {"card": card(), "map_points": int(m.num_points())}
    if args.solver != "GN":
        info["solver"] = args.solver
    print(json.dumps(info), flush=True)

    def solo_all(kps, frames):
        for k, f in zip(kps, frames):
            m.icp_register(io, k, f, prev, mm)

    def batch_all(kps, frames):
        if args.solver == "GN":
            m.icp_register_batch(io, kps, frames, [prev] * len(kps), mm)
        else:
            m.icp_register_batch_ex(io, kps, frames, [prev] * len(kps), mm)

    def host_ms(fn, kps, frames):
        for _ in range(args.warmup):
            fn([k.copy() for k in kps], [f.copy() for f in frames])
        t = []
        for _ in range(args.repeats):
            ks, fs = [k.copy() for k in kps], [f.copy() for f in frames]
            t0 = time.perf_counter()
            fn(ks, fs)
            t.append((time.perf_counter() - t0) * 1e3)
        return float(np.median(t))

    def device_ms(fn, kps, frames):
        fn([k.copy() for k in kps], [f.copy() for f in frames])   # warm
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(10):
                fn([k.copy() for k in kps], [f.copy() for f in frames])
            torch.cuda.synchronize()
        us = [e.device_time_total for e in prof.events() if kernel in e.name]
        return sum(us) / 10 / 1e3, len(us) // 10

    rows = []
    for K in (args.small, len(kp_full)):
        kp = kp_full[:K].copy()
        for B in batches:
            kps = [kp] * B
            frames = [perturbed(frame, k) for k in range(B)]
            r = {"K": K, "B": B}
            r["solo_host_ms_per_problem"] = host_ms(solo_all, kps, frames) / B
            r["batch_host_ms_per_problem"] = host_ms(batch_all, kps, frames) / B
            r["solo_device_ms"], r["solo_launches"] = device_ms(solo_all, kps, frames)
            r["batch_device_ms"], r["batch_launches"] = device_ms(batch_all, kps, frames)
            r["batch_le_solo"] = r["batch_device_ms"] <= r["solo_device_ms"]
            rows.append(r)
            print(json.dumps(r), flush=True)

    print("\n%s\n" % info["card"])
    print("| K | B | e2e solo ms/problem | e2e batch ms/problem | device solo Σ ms | device batch ms | batch/solo |")
    print("|---|---|---|---|---|---|---|")
    for r in rows:
        print("| %d | %d | %.3f | %.3f | %.3f | %.3f | %.2f |" % (
            r["K"], r["B"], r["solo_host_ms_per_problem"], r["batch_host_ms_per_problem"], r["solo_device_ms"],
            r["batch_device_ms"], r["batch_device_ms"] / max(r["solo_device_ms"], 1e-9)))
    if not all(r["batch_le_solo"] for r in rows):
        print("batched device time exceeds the sum of the solo device times at some (B, K)")
        sys.exit(1)


if __name__ == "__main__":
    main()
