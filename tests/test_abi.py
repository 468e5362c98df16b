"""CPU tests of the drop-in boundary: the engine library loads, exports every symbol include/cticp.h declares, the
ctypes mirror has the compiled struct sizes, defaults agree with the oracle's independent restatement of the
reference defaults, and a missing CUDA device is a loud error (no CPU fallback)."""
import ctypes as C
import os
import re

import pytest

import ct_icp_b200
from ct_icp_b200 import _abi as abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "cticp.h")).read()
    return sorted(set(re.findall(r"\b(cticp_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    eng = ct_icp_b200.engine()
    names = _declared_symbols()
    assert len(names) >= 35
    missing = [n for n in names if not hasattr(eng.lib, n)]
    assert not missing, missing


def test_struct_sizes_match_the_compiled_header():
    eng = ct_icp_b200.engine()
    pairs = {
        "cticp_icp_options": abi.IcpOptions, "cticp_resolution_param": abi.ResolutionParam,
        "cticp_map_options": abi.MapOptions, "cticp_strategy_options": abi.StrategyOptions,
        "cticp_motion_model_options": abi.MotionModelOptions, "cticp_odometry_options": abi.OdometryOptions,
        "cticp_pose": abi.Pose, "cticp_frame": abi.Frame, "cticp_wpoint": abi.WPoint,
        "cticp_icp_summary": abi.IcpSummary, "cticp_summary": abi.Summary, "cticp_device_timing": abi.DeviceTiming,
        "cticp_adaptive_options": abi.AdaptiveOptions,
    }
    for name, cls in pairs.items():
        assert eng.fn("abi_sizeof")(name.encode()) == C.sizeof(cls), name
    assert C.sizeof(abi.WPoint) == 64                 # slam::WPoint3D is a 64-byte record (types.h:35-60)
    import numpy as np
    assert abi.wpoint_dtype().itemsize == 64
    assert eng.fn("abi_version")() == 1


@pytest.mark.parametrize("which", ["default", "default_driving", "robust_driving", "robust_outdoor_low_inertia"])
def test_defaults_agree_with_the_oracle(orc, which):
    eng = ct_icp_b200.engine()
    a = eng.default_odometry_options() if which == "default" else eng.profile(which)
    b = orc.default_odometry_options() if which == "default" else orc.profile(which)
    assert a.to_dict() == b.to_dict()


def test_reference_default_values():
    """Spot values of include/ct_icp/ct_icp.h:60-152, odometry.h:37-133, map.h:115-125 (SURVEY Appendix B)."""
    o = ct_icp_b200.default_odometry_options()
    c = o.ct_icp_options
    assert (c.num_iters_icp, c.solver, c.max_num_residuals, c.min_num_residuals) == (5, abi.SOLVER["CERES"], -1, 100)
    assert (c.max_number_neighbors, c.min_number_neighbors, c.num_closest_neighbors) == (20, 20, 1)
    assert (c.weight_alpha, c.weight_neighborhood, c.power_planarity) == (0.9, 0.1, 2.0)
    assert (c.threshold_orientation_norm, c.threshold_translation_norm) == (1e-4, 1e-3)
    assert (c.loss_function, c.ls_max_num_iters, c.ls_num_threads, c.ls_sigma) == (abi.LOSS["CAUCHY"], 1, 16, 0.1)
    assert c.max_dist_to_plane_ct_icp == 0.3
    assert (o.init_voxel_size, o.init_sample_voxel_size, o.init_num_frames) == (0.2, 1.0, 20)
    assert (o.voxel_size, o.sample_voxel_size, o.max_distance) == (0.5, 1.5, 100.0)
    m = o.map_options
    assert m.num_resolutions == 3 and m.default_radius == 0.8
    assert [(r.resolution, r.min_distance_between_points, r.max_num_points) for r in list(m.resolutions)[:3]] == \
        [(0.2, 0.03, 50), (0.5, 0.1, 40), (1.5, 0.15, 40)]
    legacy = ct_icp_b200.engine().legacy_map_options(1.0, 20, 0.1)
    assert legacy.num_resolutions == 1 and legacy.max_frames_to_keep == 1      # src/ct_icp/map.cpp:13-29


def test_no_cpu_fallback():
    """Without a usable sm_90 device every constructor fails loudly with CTICP_ERR_NO_DEVICE."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    eng = ct_icp_b200.engine()
    with pytest.raises(ct_icp_b200.CticpError) as e:
        ct_icp_b200.Odometry(ct_icp_b200.default_odometry_options())
    assert e.value.code == abi.ERR_NO_DEVICE
    with pytest.raises(ct_icp_b200.CticpError) as e:
        ct_icp_b200.VoxelMap(eng.default_map_options())
    assert e.value.code == abi.ERR_NO_DEVICE
    import numpy as np
    with pytest.raises(ct_icp_b200.CticpError):
        eng.grid_sample_indices(np.zeros((4, 3)), 1.0)


def test_product_does_not_reference_the_oracle():
    """The engine sources and the package must not include, import or link anything under oracle/."""
    pkg = os.path.join(ROOT, "ct_icp_b200")
    offenders = []
    for d, _, files in os.walk(pkg):
        if os.path.basename(d) == "build":
            continue
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp", "Makefile")):
                txt = open(os.path.join(d, f), errors="ignore").read()
                if re.search(r"oracle/|liboracle|orc_[a-z]+\(|oracle_lib", txt) and f != "_binding.py":
                    offenders.append(os.path.join(d, f))
    assert not offenders, offenders
    out = os.popen("ldd %s" % ct_icp_b200.LIB_PATH).read()
    assert "oracle" not in out


def test_engine_permutation_matches_oracle(orc):
    # integer order contract: pure host code in both libraries
    eng = ct_icp_b200.engine()
    import numpy as np
    for n in (1, 5, 4097, 132481):
        assert np.array_equal(eng.permutation(0x5DEECE66D, (3 << 8) | 1, n), orc.permutation(0x5DEECE66D, (3 << 8) | 1, n))
