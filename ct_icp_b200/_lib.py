"""Loads the engine (ct_icp_b200/libcticp_b200.so, built by __graft_entry__.build() / csrc/Makefile).

There is no CPU fallback: a missing library raises, and creating an Odometry / VoxelMap without a usable sm_90
(H100) device fails with CTICP_ERR_NO_DEVICE.
"""
import ctypes
import os

from ._binding import Binding

_PKG = os.path.dirname(os.path.abspath(__file__))
# CTICP_ENGINE_LIB: an experiment build of the same engine (csrc/Makefile BUILD= OUT= EXTRA=), for A/B measurements
LIB_PATH = os.environ.get("CTICP_ENGINE_LIB") or os.path.join(_PKG, "libcticp_b200.so")
_engine = None


class EngineNotBuilt(RuntimeError):
    pass


def build(verbose=False):
    """nvcc -gencode arch=compute_90a,code=sm_90a … → libcticp_b200.so (cross-compiles without a GPU)."""
    import subprocess
    r = subprocess.run(["make", "-C", os.path.join(_PKG, "csrc"), "-j8"], capture_output=True, text=True)
    if verbose or r.returncode != 0:
        print(r.stdout[-4000:])
        print(r.stderr[-4000:])
    if r.returncode != 0:
        raise RuntimeError("building libcticp_b200.so failed")
    return LIB_PATH


def engine():
    """The Binding over libcticp_b200.so (prefix cticp_)."""
    global _engine
    if _engine is None:
        if not os.path.exists(LIB_PATH):
            raise EngineNotBuilt(
                f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(the engine is CUDA-only; there is no CPU fallback)")
        _engine = Binding(ctypes.CDLL(LIB_PATH), "cticp_")
    return _engine
