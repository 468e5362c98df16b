#!/usr/bin/env python
"""run_odometry -c CONFIG (command/cmd_run_odometry.cpp): runs the odometry over every sequence of the configuration's
dataset as the reference's OdometryRunner does, on the device, and writes <output_dir>[/<date>]/<sequence>.PLY and
metrics.yaml. --concurrent N (or the top-level key concurrent_sequences: N) registers up to N sequences side by side in
one batched call per frame; the files are those of the serial run, up to summation order when the batch's problems do
not fit on the device together. Exits 1 when a frame failed with exit_early.
usage: python tools/run_odometry.py -c config.yaml [--concurrent N] [--device 0]"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import ct_icp_b200  # noqa: E402
from ct_icp_b200 import config, datasets, runner  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser(description="Runs the CT-ICP odometry on all sequences of the configured dataset")
    ap.add_argument("-c", "--config", required=True, help="path to the YAML configuration")
    ap.add_argument("--concurrent", type=int, default=None, help="sequences registered side by side (default: the "
                    "config's concurrent_sequences, else 1)")
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args(argv)
    b = ct_icp_b200.engine()
    root = config.load_config(args.config)
    dataset_options = config.dataset_options_from_config(root)
    options = config.load_runner_options(root, b)
    if args.concurrent is not None:
        if not 1 <= args.concurrent <= 64:
            ap.error("--concurrent must be in [1, 64]")
        options.concurrent_sequences = args.concurrent
    for w in options.warnings:
        print("WARNING:", w, file=sys.stderr)
    sequences = datasets.load_dataset_from_options(b, dataset_options, device=args.device)
    for label, seq in sequences:
        print("Name: %s, Num Frames=%d" % (label, seq.NumFrames()), file=sys.stderr)
    r = runner.OdometryRunner(b, sequences, options, device=args.device, log=lambda m: print(m, file=sys.stderr))
    ok = r.Run()
    if r.output_path:
        print("outputs in", os.path.abspath(r.output_path))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
