"""ct_icp_b200 — H100-native CT-ICP registration engine behind the ct_icp::Odometry API surface.

Python host mirror of the reference interface (ct_icp::Odometry, CTICPOptions, OdometryOptions,
MultipleResolutionVoxelMap) over the C ABI in include/cticp.h. All compute runs in hand-written sm_90a kernels
(ct_icp_b200/csrc); this package only marshals arrays and option structs.
"""
from . import _abi as abi
from ._binding import CticpError
from ._lib import LIB_PATH, EngineNotBuilt, build, engine


def default_odometry_options():
    """ct_icp::OdometryOptions() defaults (include/ct_icp/odometry.h:37-157)."""
    return engine().default_odometry_options()


def profile(name):
    """OdometryOptions::DefaultDrivingProfile / RobustDrivingProfile / DefaultRobustOutdoorLowInertia
    → name in {"default_driving", "robust_driving", "robust_outdoor_low_inertia"}."""
    return engine().profile(name)


def Odometry(options, device=0):
    """ct_icp::Odometry(options) on CUDA device `device`."""
    return engine().odometry(options, device)


def VoxelMap(options, device=0):
    """ct_icp::MultipleResolutionVoxelMap(options) on CUDA device `device`."""
    return engine().voxel_map(options, device)


__all__ = ["abi", "CticpError", "EngineNotBuilt", "LIB_PATH", "build", "engine", "default_odometry_options",
           "profile", "Odometry", "VoxelMap"]
