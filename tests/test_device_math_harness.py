"""The device-math harness (tests/cuda/device_math.cu) compiles against the current csrc headers with the library's
NVFLAGS (nvcc cross-compiles for sm_90a without a GPU): a header change that breaks a routine's signature or the
harness's use of it fails here, not only on the GPU machine. CPU only."""
import ctypes
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ["sym_eig3", "describe", "ldlt_solve12", "gn_solve", "ct_residual", "dq_dot", "quat_plus", "loss_evaluate",
           "corrector", "ct_transform", "qfromR", "qtoR", "voxel_coord_rcp"]


def test_device_math_harness_compiles(tmp_path):
    out = tmp_path / "libcticp_device_math.so"
    r = subprocess.run(["make", "-C", os.path.join(ROOT, "ct_icp_b200", "csrc"), "device_math", "DM_OUT=%s" % out,
                        "BUILD=%s" % (tmp_path / "build")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "-O3" in r.stdout and "arch=compute_90a,code=sm_90a" in r.stdout   # the library's flags, verbatim
    lib = ctypes.CDLL(str(out))   # loads without a device: no CUDA call runs at load time
    for e in ENTRIES:
        assert hasattr(lib, "dm_" + e), e
