"""csrc/cuda_owner.h (the owners of the engine's CUDA buffers, streams and events) built with plain g++ against the
static CUDA runtime. Without a usable device every allocation fails: reserve throws a CudaError naming the call and
leaves the holder empty, so the next reserve allocates again. With a device: growth, reuse of a large enough
allocation, and moves that leave the source empty."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = "/usr/local/cuda"


def test_cuda_owner(tmp_path):
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "cuda_owner_test")
    r = subprocess.run([cxx, "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(CUDA, "include"), "-I",
                        os.path.join(ROOT, "ct_icp_b200", "csrc"), os.path.join(ROOT, "tests", "cpp", "cuda_owner_test.cpp"),
                        "-L", os.path.join(CUDA, "lib64"), "-lcudart_static", "-ldl", "-lpthread", "-lrt", "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "CUDA OWNER OK" in r.stdout, r.stdout + r.stderr
