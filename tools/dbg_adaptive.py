import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
from oracle_lib import oracle
import ct_icp_b200
from ct_icp_b200 import _abi as abi, synthetic as syn
from test_gpu_parity import nclt_config
from conftest import frame_diff
orc=oracle(); eng=ct_icp_b200.engine()
seq = syn.make_sequence(3, syn.HDL32, seed=78, traj=syn.Trajectory(speed=2.0, sway=1.0, sway_rate=0.2, height=1.0))
ods=[]
for b in (orc,eng):
    o=nclt_config(b, "CERES"); o.sampling=abi.SAMPLING["ADAPTIVE"]
    o.ct_icp_options.num_iters_icp = int(sys.argv[1]); o.ct_icp_options.ls_max_num_iters=int(sys.argv[2]); o.ct_icp_options.ls_num_threads=1
    ods.append(b.odometry(o))
for i,s in enumerate(seq):
    if i==2:
        os.environ["ORC_DEBUG_LM"]="1"; os.environ["CTICP_DEBUG_LM"]="1"
    so=ods[0].RegisterFrame(s["xyz"],s["t"],s["frame_idx"]); se=ods[1].RegisterFrame(s["xyz"],s["t"],s["frame_idx"])
    print(i,"diff",frame_diff(so.frame,se.frame), "iters", so.icp_summary.num_iters, se.icp_summary.num_iters)
