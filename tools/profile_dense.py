import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench, ct_icp_b200
from ct_icp_b200 import synthetic as syn
bench._WORKLOAD="dense128_gn"
eng=ct_icp_b200.engine()
seq=syn.make_sequence(8, syn.DENSE128, seed=1234)
od=eng.odometry(bench.make_options(eng))
slots=[od.stage_frame(s["xyz"],s["t"]) for s in seq]
for i,s in enumerate(seq):
    sm=od.RegisterStaged(slots[i], s["frame_idx"]); t=od.last_timing()
    print(i, "launches",t.kernel_launches,"total %.3f ingest %.3f icp %.3f map %.3f"%(t.total_ms,t.ingest_ms,t.icp_ms,t.map_update_ms),"K",sm.num_keypoints,"F",sm.num_corrected_points, "iters", sm.icp_summary.num_iters)
print("--- with L2 flush + stopwatch (bench protocol)")
od2 = eng.odometry(bench.make_options(eng))
slots2 = [od2.stage_frame(s["xyz"], s["t"]) for s in seq]
for i, s in enumerate(seq):
    od2.flush_l2(256 << 20)
    od2.timer_start()
    sm = od2.RegisterStaged(slots2[i], s["frame_idx"])
    ms = od2.timer_stop()
    t = od2.last_timing()
    print(i, "stopwatch %.3f ms" % ms, "total %.3f ingest %.3f icp %.3f map %.3f" % (t.total_ms, t.ingest_ms, t.icp_ms, t.map_update_ms))
