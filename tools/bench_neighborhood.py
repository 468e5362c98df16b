"""Neighbourhood benchmark: the k-nearest index (cticp_neighborhood_*) over world clouds of the lidar scans of
tools/bench_world_cloud.py, against scipy.spatial.cKDTree(workers=-1) on the same points on this host.

Workloads: a world cloud of --scans[0] scans at 0.1 m: build, self-search and self-describe with k 10 and 20, unbounded
and with max_radius 0.25 (a 0.5 m radius); --scans[1] scans: k 20 self-describe; 1M queries spread over the cloud's
bounding box grown by 50 m. Timings are CUDA events around synchronised work after one untimed pass over the same
shapes, with the queries and outputs in device memory (the device variants: the host variants add the copies of
the m x k outputs). cKDTree's neighbour sets are checked on a sample (ties are the only allowed difference). One JSON line each.

python tools/bench_neighborhood.py [--scans 64 512] [--cpu-sample 200000]
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
sys.path.insert(0, os.path.join(ROOT, "tools"))


def world(eng, torch, S):
    from bench_world_cloud import PER_SCAN, frames, make_scans
    traj = eng.continuous_trajectory(frames(S))
    xyz, t = make_scans(torch, S, 1)
    wc = eng.world_cloud(0.1, 1, capacity_voxels=1 << 26)
    for k in range(S):
        wc.add(xyz[k * PER_SCAN:(k + 1) * PER_SCAN], t[k * PER_SCAN:(k + 1) * PER_SCAN], traj)
    return wc


def timed(torch, fn, reps=1):
    fn()   # warm-up over the same shapes
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, nargs="+", default=[64, 512])
    ap.add_argument("--cpu-sample", type=int, default=200000)
    args = ap.parse_args()
    import torch
    from scipy.spatial import cKDTree

    import ct_icp_b200
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU only")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps({"gpu": smi}), flush=True)
    eng = ct_icp_b200.engine()

    def emit(**kw):
        print(json.dumps(kw), flush=True)

    for wi, S in enumerate(args.scans):
        wc = world(eng, torch, S)
        pts = wc.export()
        qd = wc.export(device=True)   # the indexed points as device queries: the self queries of the device variant
        n = len(pts)
        ms, nb = timed(torch, lambda: wc.neighborhood())
        emit(workload="build", scans=S, points=n, ms=round(ms, 3))
        cases = [(10, None), (20, None), (10, 0.25), (20, 0.25)] if wi == 0 else [(20, None)]
        for k, r in cases:
            rad = np.finfo(np.float64).max if r is None else r
            for op in (("search", "describe") if wi == 0 else ("describe",)):
                fn = (lambda: nb.search(qd, k, rad)) if op == "search" else (lambda: nb.describe(qd, k, rad))
                ms, _ = timed(torch, fn)
                emit(workload="self_" + op, scans=S, points=n, k=k, max_radius=r, ms=round(ms, 2),
                     mquery_s=round(n / ms / 1e3, 2))
        if wi == 0:
            rng = np.random.default_rng(0)
            lo, hi = pts.min(0) - 50, pts.max(0) + 50
            q = rng.uniform(lo, hi, (1_000_000, 3))
            qb = torch.tensor(q, device="cuda")
            ms, _ = timed(torch, lambda: nb.search(qb, 20))
            emit(workload="box_queries", points=n, queries=len(q), k=20, ms=round(ms, 2), mquery_s=round(len(q) / ms / 1e3, 3))
            # cKDTree on the same points, this host, all cores
            t0 = time.perf_counter()
            tree = cKDTree(pts)
            tb = time.perf_counter() - t0
            sample = rng.integers(0, n, min(args.cpu_sample, n))
            t0 = time.perf_counter()
            dd, ii = tree.query(pts[sample], k=20, workers=-1)
            tq = time.perf_counter() - t0
            emit(workload="ckdtree", points=n, build_s=round(tb, 3), k=20, queries=len(sample),
                 mquery_s=round(len(sample) / tq / 1e6, 3), cpus=os.cpu_count())
            t0 = time.perf_counter()   # a NumPy statement of the descriptors of those neighbourhoods
            nbh = pts[ii]
            c = nbh - nbh.mean(1, keepdims=True)
            cov = np.einsum("qki,qkj->qij", c, c) / 20
            w, v = np.linalg.eigh(cov)
            tn = time.perf_counter() - t0
            emit(workload="numpy_describe", queries=len(sample), mquery_s=round(len(sample) / tn / 1e6, 3))
            gi, gd, gc = nb.search(pts[sample], 20)
            agree = 0
            for j in range(len(sample)):
                if set(gi[j].tolist()) == set(ii[j].tolist()):
                    agree += 1
                else:   # only ties at the k-th distance may differ
                    assert np.isclose(gd[j, -1], dd[j, -1] ** 2, rtol=1e-12), j
            emit(workload="ckdtree_agreement", sample=len(sample), identical_sets=agree)
        del nb, wc, qd
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
