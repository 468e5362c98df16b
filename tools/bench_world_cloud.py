"""World-cloud benchmark: grid-sampling S synthetic 130k-point scans along a trajectory into one device-resident cloud
(cticp_world_cloud_*), against the CPU path that exists without it (cticp_trajectory_transform to host, then a NumPy
grid sample).

For each (scans, grid, num_points_per_voxel): add throughput of the device input (torch CUDA tensors, one add per scan),
of the host input (NumPy records, one add per scan, copies included), export time (device, fp64 xyz + t + source
index), and once per grid the odometry input (add_odometry of a registered synthetic scan). Every timing is CUDA
events around synchronised work, after one untimed pass over the same shapes; each configuration is run --repeat times.
The export of every timed run is checked against the CPU restatement (tests/oracle_grid) over the concatenated world
points. Prints one JSON line per measurement.

python tools/bench_world_cloud.py [--scans 64 512] [--grids 0.1 0.2] [--npv 1 4] [--repeat 3] [--cpu-scans 64]
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

PER_SCAN = 130_000


def frames(n):
    from ct_icp_b200 import _abi as abi
    out = []
    for k in range(n):
        f = abi.Frame()
        yaw0, yaw1 = 0.01 * k, 0.01 * (k + 1)
        f.begin_pose = abi.Pose.make(quat=[0, 0, np.sin(yaw0 / 2), np.cos(yaw0 / 2)], tr=[1.0 * k, 0.02 * k, 0.0],
                                     dest_timestamp=0.1 * k, dest_frame_id=k)   # boundaries shared exactly
        f.end_pose = abi.Pose.make(quat=[0, 0, np.sin(yaw1 / 2), np.cos(yaw1 / 2)], tr=[1.0 * k + 1.0, 0.02 * k + 0.02, 0.0],
                                   dest_timestamp=0.1 * (k + 1), dest_frame_id=k)
        out.append(f)
    return out


def make_scans(torch, n_scans, seed):
    """lidar-like raw scans: 64 rings at elevations -25..+3 degrees hitting a ground plane 1.7 m below or a cylinder
    wall at 5-60 m; float32 (N, 4) xyzi, timestamps over the frame"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = n_scans * PER_SCAN
    az = torch.rand(n, generator=g, device="cuda", dtype=torch.float64) * 2 * np.pi
    el = torch.deg2rad(-25.0 + 28.0 * torch.randint(0, 64, (n,), generator=g, device="cuda").double() / 63.0)
    wall = 5.0 + 55.0 * torch.rand(n, generator=g, device="cuda", dtype=torch.float64)
    r_ground = torch.where(el < -0.02, 1.7 / torch.tan(-el).clamp(min=1e-3), torch.full_like(el, 1e9))
    r = torch.minimum(wall / torch.cos(el), r_ground)
    xyz = torch.empty((n, 4), dtype=torch.float32, device="cuda")
    xyz[:, 0] = (r * torch.cos(el) * torch.cos(az)).float()
    xyz[:, 1] = (r * torch.cos(el) * torch.sin(az)).float()
    xyz[:, 2] = (r * torch.sin(el)).float()
    xyz[:, 3] = 0.0
    fr = torch.arange(n, device="cuda") // PER_SCAN
    t = 0.1 * fr.double() + 0.1 * az / (2 * np.pi)
    return xyz, t


def timed(torch, fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, nargs="+", default=[64, 512])
    ap.add_argument("--grids", type=float, nargs="+", default=[0.1, 0.2])
    ap.add_argument("--npv", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--cpu-scans", type=int, default=64)
    args = ap.parse_args()

    import torch
    import ct_icp_b200
    from grid_numpy import sample_points_in_grid as np_sample
    from oracle_grid_lib import grid_oracle

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU only")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps({"gpu": smi}), flush=True)
    eng = ct_icp_b200.engine()
    orc = grid_oracle()
    smax = max(args.scans)
    traj = eng.continuous_trajectory(frames(smax))
    xyz, t = make_scans(torch, smax, 1)
    for S in args.scans:
        n = S * PER_SCAN
        world = traj.transform(xyz[:n], t[:n], dtype=np.float64).cpu().numpy()   # the check's input
        for grid in args.grids:
            for npv in args.npv:
                ref = orc.sample_points_in_grid(world, grid, npv)
                wc = eng.world_cloud(grid, npv, capacity_voxels=len(ref) + 1, capacity_points=len(ref) + 1)
                xs = [xyz[k * PER_SCAN:(k + 1) * PER_SCAN] for k in range(S)]
                ts = [t[k * PER_SCAN:(k + 1) * PER_SCAN] for k in range(S)]
                xh = [x[:, :3].cpu().numpy() for x in xs]
                th = [x.cpu().numpy() for x in ts]

                def dev_run():
                    for x, tt in zip(xs, ts):
                        wc.add(x, tt, trajectory=traj)

                def host_run():
                    for x, tt in zip(xh, th):
                        wc.add(x, tt, trajectory=traj)

                def export():
                    return wc.export(np.float64, with_timestamps=True, with_source_index=True, device=True)

                for name, run in (("device", dev_run), ("host", host_run)):
                    wc.clear()
                    run()                       # warm-up: every shape of the timed window
                    export()
                    for rep in range(args.repeat):
                        wc.clear()
                        ms, _ = timed(torch, run)
                        ems, (pts, src) = timed(torch, export)
                        ok = np.array_equal(src.cpu().numpy().astype(np.uint64), ref)
                        print(json.dumps({"input": name, "scans": S, "points": n, "grid": grid, "npv": npv, "rep": rep,
                                          "add_ms": round(ms, 3), "mpoint_s": round(n / ms / 1e3, 1),
                                          "export_ms": round(ems, 3), "kept": int(pts.shape[0]),
                                          "voxels": wc.num_voxels(), "matches_restatement": ok}), flush=True)
                        if not ok:
                            raise SystemExit("export differs from the restatement")
                wc.close()
                if S == args.cpu_scans:
                    # the path without a world cloud: transform to host, then grid-sample the concatenation in NumPy
                    for rep in range(args.repeat):
                        t0 = time.perf_counter()
                        w = traj.transform(xyz[:n, :3].cpu().numpy(), t[:n].cpu().numpy(), dtype=np.float64)
                        idx = np_sample(w, grid, npv)
                        dt = (time.perf_counter() - t0) * 1e3
                        print(json.dumps({"input": "cpu_numpy", "scans": S, "points": n, "grid": grid, "npv": npv,
                                          "rep": rep, "total_ms": round(dt, 1), "mpoint_s": round(n / dt / 1e3, 2),
                                          "matches_restatement": bool(np.array_equal(idx, ref))}), flush=True)
    # odometry input: add_odometry of a registered synthetic scan (its ALL_CORRECTED points), repeated
    from ct_icp_b200 import _abi as abi
    from ct_icp_b200 import synthetic as syn
    o = eng.default_odometry_options()
    o.ct_icp_options.solver = abi.SOLVER["GN"]
    o.ct_icp_options.min_number_neighbors = 10
    o.map_options = eng.legacy_map_options(1.0, 20, 0.1)
    o.init_num_frames = 3
    o.debug_print = 0
    o.ct_icp_options.debug_print = 0
    od = eng.odometry(o)
    for s in syn.make_sequence(4, syn.SMALL16, seed=7):
        assert od.RegisterFrame(s["xyz"], s["t"], s["frame_idx"]).success
    m = od.points_device(abi.POINTS_ALL_CORRECTED).shape[0]
    for grid in args.grids:
        wc = eng.world_cloud(grid, 4)
        wc.add_odometry(od)
        for rep in range(args.repeat):
            wc.clear()
            ms, _ = timed(torch, lambda: [wc.add_odometry(od) for _ in range(64)])
            print(json.dumps({"input": "odometry", "points": 64 * m, "adds": 64, "grid": grid, "npv": 4, "rep": rep,
                              "add_ms": round(ms, 3), "mpoint_s": round(64 * m / ms / 1e3, 1)}), flush=True)
        wc.close()
    od.close()


if __name__ == "__main__":
    main()
