#!/usr/bin/env python
"""The reference's odometry runner loop (command/odometry_runner.cpp) over one dataset sequence, on the device: every
frame is read and filtered on the GPU (ct_icp_b200.datasets), registered with Odometry.register_device, and its end pose
written in KITTI format as SavePosesKITTIFormat writes it (io.cxx:282-304). With ground truth, the estimate is scored
with ComputeTrajectoryMetrics (cticp_trajectory_metrics) against the ground truth at the frames' end timestamps and the
scores printed as one JSON line. --out-ply writes the runner's <sequence>.PLY as SaveTrajectoryAndMetrics does
(odometry_runner.cpp:318-340, save_mid_frame false): the first frame's begin pose, then every frame's end pose, through
SavePosesAsPLY.
usage: python tools/run_sequence.py --dataset NCLT --root DIR --sequence 2012-01-08 --out poses.txt
       [--out-ply poses.PLY] [--max-frames N] [--init-frame K] [--device 0]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

import ct_icp_b200  # noqa: E402
from ct_icp_b200 import _abi as abi  # noqa: E402
from ct_icp_b200 import datasets  # noqa: E402


def kitti_lines(poses):
    """SavePosesKITTIFormat: R | t row by row, 17 significant digits"""
    from scipy.spatial.transform import Rotation
    out = []
    for p in poses:
        q = np.array(p.quat[:])
        R = Rotation.from_quat(q / np.linalg.norm(q)).as_matrix()
        t = p.tr[:]
        vals = [R[0, 0], R[0, 1], R[0, 2], t[0], R[1, 0], R[1, 1], R[1, 2], t[1], R[2, 0], R[2, 1], R[2, 2], t[2]]
        out.append(" ".join("%.17g" % v for v in vals))
    return out


def run(binding, sequence, options, device=0, begin_poses=None):
    """register every frame of `sequence`; returns the end poses, the frames' end timestamps and whether every frame
    registered; each frame's begin pose is appended to `begin_poses` when given"""
    import torch
    od = binding.odometry(options, device=device)
    stream = torch.cuda.current_stream(device).cuda_stream
    poses, stamps, ok = [], [], True
    while sequence.HasNext():
        frame = sequence.NextFrame()
        sm = od.register_device(datasets.device_scan(frame), frame["frame_id"], stream=stream)
        ok = ok and bool(sm.success)
        if begin_poses is not None:
            begin_poses.append(sm.frame.begin_pose)
        poses.append(sm.frame.end_pose)
        stamps.append(float(frame["t"].max().item()) if frame["t"].numel() else float("nan"))
    return poses, np.array(stamps), ok


def score(binding, sequence, poses, stamps, device=0):
    """the estimate against the ground truth interpolated at the frames' end timestamps, both taken relative to their
    first pose; None without ground truth"""
    gt = sequence.GroundTruth()
    if gt is None or len(gt) == 0 or len(poses) < 2:
        return None
    g = binding.continuous_trajectory(datasets.pose_list(gt), device=device).interpolate(stamps)
    gt_rel, est_rel = [], []
    q0g, t0g = np.array(g[0]["quat"]), np.array(g[0]["tr"])
    from scipy.spatial.transform import Rotation
    R0g = Rotation.from_quat(q0g / np.linalg.norm(q0g))
    q0e, t0e = np.array(poses[0].quat[:]), np.array(poses[0].tr[:])
    R0e = Rotation.from_quat(q0e / np.linalg.norm(q0e))
    for k in range(len(poses)):
        qg, tg = np.array(g[k]["quat"]), np.array(g[k]["tr"])
        qe, te = np.array(poses[k].quat[:]), np.array(poses[k].tr[:])
        rg = R0g.inv() * Rotation.from_quat(qg / np.linalg.norm(qg))
        re = R0e.inv() * Rotation.from_quat(qe / np.linalg.norm(qe))
        gt_rel.append(abi.Pose.make(rg.as_quat().tolist(), R0g.inv().apply(tg - t0g).tolist(), float(k), k))
        est_rel.append(abi.Pose.make(re.as_quat().tolist(), R0e.inv().apply(te - t0e).tolist(), float(k), k))
    ape = max(float(np.linalg.norm(np.array(a.tr[:]) - np.array(b.tr[:]))) for a, b in zip(gt_rel, est_rel))
    out = {"max_ape_m": ape, "mean_ate": None, "max_ate": None}
    if len(poses) >= 5:   # ComputeTrajectoryMetrics needs five poses
        m = binding.trajectory_metrics(gt_rel, est_rel, segment_length=10.0, device=device)
        out["mean_ate"], out["max_ate"] = float(m["mean_ate"]), float(m["max_ate"])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dataset", required=True, choices=sorted(abi.DATASET))
    ap.add_argument("--root", required=True)
    ap.add_argument("--sequence", required=True)
    ap.add_argument("--out", required=True)
    ap.add_argument("--out-ply", default=None)
    ap.add_argument("--max-frames", type=int, default=-1)
    ap.add_argument("--init-frame", type=int, default=0)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    b = ct_icp_b200.engine()
    seqs = datasets.load_dataset(b, args.dataset, args.root, [args.sequence], device=args.device)
    if not seqs:
        sys.exit("no sequence %s of %s under %s" % (args.sequence, args.dataset, args.root))
    seq = seqs[0][1]
    seq.SetInitFrame(args.init_frame)
    seq.SetMaxNumFrames(args.max_frames)
    o = b.default_odometry_options()
    begins = []
    poses, stamps, ok = run(b, seq, o, args.device, begins)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write("\n".join(kitti_lines(poses)) + "\n")
    if args.out_ply:
        os.makedirs(os.path.dirname(os.path.abspath(args.out_ply)), exist_ok=True)
        with open(args.out_ply, "wb") as f:
            f.write(b.save_poses_ply(begins[:1] + poses, device=args.device))
    print(json.dumps({"frames": len(poses), "success": ok, "scores": score(b, seq, poses, stamps, args.device)}))


if __name__ == "__main__":
    main()
