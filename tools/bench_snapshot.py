"""Snapshot cost on one GPU: the size of an odometry snapshot, the pack / unpack kernel times (torch.profiler, device
events) with their bytes/s against the H100's 3.35 TB/s, and the wall time of save, load, clone and of creating a
handle with the same options (median, min, max), after one warm-up load and clone.

Maps: the GN bench options on an HDL-64 sequence after 60 frames (the kitti64_gn pre-roll of 20 plus 40), and on a
DENSE-128 sequence after 20 frames. Prints one JSON line per map, with the card name and power limit of this run.

    python tools/bench_snapshot.py [--frames-hdl64 60] [--frames-dense128 20] [--repeats 5]
"""
import argparse
import ctypes as C
import json
import os
import struct
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import ct_icp_b200  # noqa: E402
from ct_icp_b200 import _abi as abi  # noqa: E402
from ct_icp_b200 import synthetic as syn  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12
HEADER = 72   # snapshot_format.h kHeaderBytes


def gn_options(eng):
    o = eng.default_odometry_options()
    o.ct_icp_options.solver = abi.SOLVER["GN"]
    o.ct_icp_options.num_iters_icp = 5
    o.ct_icp_options.min_number_neighbors = 10
    o.map_options = eng.legacy_map_options(1.0, 20, 0.1)
    o.voxel_size, o.sample_voxel_size, o.max_distance = 0.5, 1.5, 100.0
    o.debug_print = 0
    o.ct_icp_options.debug_print = 0
    return o


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def kernel_us(fn, name):
    """device time of the kernels whose name contains `name` during fn(), in µs (torch.profiler)"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    total = 0.0
    for e in prof.events():
        if name in e.name and e.device_type.name == "CUDA":
            total += e.device_time if hasattr(e, "device_time") else e.cuda_time
    return total


def map_bytes(blob):
    """(slot-table bytes, map payload bytes) of an odometry snapshot: the level headers of its map section
    (snapshot_format.h)"""
    sizes = struct.unpack_from("<5Q", blob, 16)
    at = HEADER + sum(sizes[:3])
    levels = struct.unpack_from("<I", blob, at + C.sizeof(abi.MapOptions))[0]
    table = sum(16 * struct.unpack_from("<Q", blob, at + C.sizeof(abi.MapOptions) + 16 + 48 * i)[0] for i in range(levels))
    header = C.sizeof(abi.MapOptions) + 16 + 48 * levels
    return table, sizes[3] - header


def measure(eng, label, sensor, frames, repeats):
    od = eng.odometry(gn_options(eng))
    for s in syn.make_sequence(frames, sensor, seed=1234):
        od.RegisterFrame(s["xyz"], s["t"], s["frame_idx"])
    blob = od.save()
    m = od.GetMapPointer()
    res = {"map": label, "frames": frames, "points": m.num_points(0), "voxels": m.num_voxels(0), "snapshot_bytes": len(blob)}
    # One byte count for both kernels: the pack reads every slot of the tables and the live runs and writes the packed
    # records, runs and normals (table + 2 x payload); the unpack reads the packed payload and writes the same records
    # and runs into their slots (2 x payload). The tables it writes were cleared before, by k_clear_level.
    table, payload = map_bytes(blob)
    pack_bytes, unpack_bytes = table + 2 * payload, 2 * payload
    eng.load_odometry(blob).close()   # warm-up: the first load and clone of the process pay one-time costs
    od.clone().close()
    pack = [kernel_us(od.save, "k_snapshot_pack") for _ in range(repeats)]
    unpack = [kernel_us(lambda: eng.load_odometry(blob).close(), "k_snapshot_unpack") for _ in range(repeats)]
    res["table_bytes"], res["payload_bytes"] = table, payload
    res["pack_us"] = float(np.median(pack))
    res["unpack_us"] = float(np.median(unpack))
    res["pack_GBps"] = pack_bytes / (res["pack_us"] * 1e-6) / 1e9
    res["unpack_GBps"] = unpack_bytes / (res["unpack_us"] * 1e-6) / 1e9
    res["pack_frac_of_peak"] = res["pack_GBps"] * 1e9 / PEAK_BYTES_PER_S
    res["unpack_frac_of_peak"] = res["unpack_GBps"] * 1e9 / PEAK_BYTES_PER_S

    def wall(fn):
        ts = []
        for _ in range(repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            ts.append((time.perf_counter() - t0) * 1e3)
        return float(np.median(ts)), float(min(ts)), float(max(ts))

    res["save_ms"] = wall(od.save)
    res["load_ms"] = wall(lambda: eng.load_odometry(blob).close())
    res["clone_ms"] = wall(lambda: od.clone().close())
    # what load and clone build besides the map: a new handle with the same options, created and destroyed
    res["new_handle_ms"] = wall(lambda: eng.odometry(gn_options(eng)).close())
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames-hdl64", type=int, default=60)
    ap.add_argument("--frames-dense128", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    eng = ct_icp_b200.engine()
    name, power = card()
    for label, sensor, frames in (("kitti64_gn", syn.HDL64, a.frames_hdl64), ("dense128_gn", syn.DENSE128, a.frames_dense128)):
        r = measure(eng, label, sensor, frames, a.repeats)
        r["gpu"], r["power_limit"] = name, power
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
