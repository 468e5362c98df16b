"""Target of the compute-sanitizer runs (tools/gpu_sanitize.sh): a short odometry sequence through the C ABI for one
solver, every round-2 kernel on the path (fused sampler, persistent GN / LM kernel with its grid barriers, selection with
shared-memory staging, fused map update, egress stream). Exits non-zero if a registration fails."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import ct_icp_b200  # noqa: E402
from ct_icp_b200 import _abi as abi  # noqa: E402
from ct_icp_b200 import synthetic as syn  # noqa: E402

solver = sys.argv[1] if len(sys.argv) > 1 else "GN"
frames = int(sys.argv[2]) if len(sys.argv) > 2 else 5
eng = ct_icp_b200.engine()
o = eng.default_odometry_options()
o.ct_icp_options.solver = abi.SOLVER[solver]
o.ct_icp_options.min_number_neighbors = 10
o.ct_icp_options.ls_max_num_iters = 3
o.map_options = eng.legacy_map_options(1.0, 20, 0.1)
o.map_options.capacity_voxels = 1 << 14
o.init_num_frames = 2
o.debug_print = 0
od = eng.odometry(o)
od.set_summary_points(7)
for s in syn.make_sequence(frames, syn.SMALL16, seed=1234):
    sm = od.RegisterFrame(s["xyz"], s["t"], s["frame_idx"])
    assert sm.success, sm.error_message
    n = len(od.all_corrected_points())
    print(s["frame_idx"], "K", sm.num_keypoints, "residuals", sm.number_of_residuals, "points", n, flush=True)
if solver == "GN":
    # batched GN (k_gn_persistent over groups): three small problems against the odometry's map, the last one failing
    # with fewer than 100 residuals
    kp = od.keypoints()
    frame = od.Trajectory()[-1]
    kps = [kp[:200].copy(), kp[200:400].copy(), kp[:50].copy()]
    io = o.ct_icp_options.copy()
    io.num_iters_icp = 4
    ss = od.GetMapPointer().icp_register_batch(io, kps, [frame.copy() for _ in kps])
    assert not ss[2].success
    print("batch", [(s.success, s.num_residuals_used, s.num_iters) for s in ss], flush=True)
od.close()
print("sanitize target OK", solver)
