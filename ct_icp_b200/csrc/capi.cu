// capi.cu — extern "C" entry points declared in include/cticp.h. No exceptions cross this boundary: every call
// returns a cticp_status and records its message for cticp_last_error().
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/cticp.h"
#include "dataset.h"
#include "engine.h"
#include "lidar_sim.h"
#include "neighborhood.h"
#include "ply.h"
#include "synthetic.h"
#include "trajectory.h"
#include "trajectory_eval.h"
#include "world_cloud.h"

using namespace cticp;

namespace {
thread_local std::string g_last_error;

int Fail(int code, const std::string &msg) {
    g_last_error = msg;
    return code;
}
template <typename F>
int Guard(F &&f) {
    try {
        return f();
    } catch (const TimestampError &e) {
        return Fail(CTICP_ERR_TIMESTAMP, e.what());
    } catch (const UnsupportedError &e) {
        return Fail(CTICP_ERR_UNSUPPORTED, e.what());
    } catch (const CapacityError &e) {
        return Fail(CTICP_ERR_CAPACITY, e.what());
    } catch (const cticp::CallbackError &e) {
        return Fail(CTICP_ERR_CALLBACK, e.what());
    } catch (const CudaError &e) {
        return Fail(CTICP_ERR_CUDA, e.what());
    } catch (const std::invalid_argument &e) {
        return Fail(CTICP_ERR_INVALID_ARGUMENT, e.what());
    } catch (const std::runtime_error &e) {
        if (std::string(e.what()).rfind("NCCL", 0) == 0) return Fail(CTICP_ERR_NCCL, e.what());
        if (std::string(e.what()).rfind("NO_DEVICE", 0) == 0) return Fail(CTICP_ERR_NO_DEVICE, e.what());
        return Fail(CTICP_ERR_INTERNAL, e.what());
    } catch (const std::exception &e) {
        if (std::string(e.what()).rfind("NO_DEVICE", 0) == 0) return Fail(CTICP_ERR_NO_DEVICE, e.what());
        return Fail(CTICP_ERR_INTERNAL, e.what());
    }
}
void RequireDevice(int device) {
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count)
        throw std::runtime_error("NO_DEVICE: no usable CUDA device (this engine has no CPU fallback)");
    CT_CUDA_CHECK(cudaSetDevice(device));
    cudaDeviceProp prop;
    CT_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) throw std::runtime_error("NO_DEVICE: this build targets sm_90a (Hopper H100) only");
}
// RequireDevice without cudaGetDeviceProperties (milliseconds per call): for the per-frame dataset entry points
void RequireDeviceCheap(int device) {
    int count = 0, major = 0, minor = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count)
        throw std::runtime_error("NO_DEVICE: no usable CUDA device (this engine has no CPU fallback)");
    CT_CUDA_CHECK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
    CT_CUDA_CHECK(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device));
    if (major != 9 || minor != 0) throw std::runtime_error("NO_DEVICE: this build targets sm_90a (Hopper H100) only");
}
}  // namespace

struct cticp_map {
    // a handle of cticp_map_create owns its stream, map and solver; an odometry's view borrows its engine's
    cticp::Stream owned_stream;
    std::unique_ptr<DeviceMap> owned_map;
    std::unique_ptr<IcpSolver> owned_icp;
    DeviceMap *map = nullptr;
    IcpSolver *icp = nullptr;
    cudaStream_t stream = nullptr;
    int device = 0;
    bool owned = false;
};
struct cticp_odometry {
    std::unique_ptr<Engine> engine;
    cticp_map map_view;
};
struct cticp_trajectory {
    std::unique_ptr<ContinuousTrajectory> impl;
};
struct cticp_world_cloud {
    std::unique_ptr<WorldCloud> impl;
};
struct cticp_neighborhood {
    std::unique_ptr<NeighborhoodIndex> impl;
};
struct cticp_synthetic_scene {
    std::unique_ptr<SyntheticScene> impl;
};
struct cticp_lidar_scene {
    std::unique_ptr<LidarScene> impl;
};
struct cticp_nclt {
    std::unique_ptr<NcltHits> impl;
};

extern "C" {

uint32_t cticp_abi_version(void) { return CTICP_ABI_VERSION; }
const char *cticp_last_error(void) { return g_last_error.c_str(); }

size_t cticp_abi_sizeof(const char *name) {
    const std::string s(name ? name : "");
    if (s == "cticp_icp_options") return sizeof(cticp_icp_options);
    if (s == "cticp_resolution_param") return sizeof(cticp_resolution_param);
    if (s == "cticp_map_options") return sizeof(cticp_map_options);
    if (s == "cticp_grid_sampling_options") return sizeof(cticp_grid_sampling_options);
    if (s == "cticp_world_cloud_stats") return sizeof(cticp_world_cloud_stats);
    if (s == "cticp_neighborhood_description") return sizeof(cticp_neighborhood_description);
    if (s == "cticp_synthetic_frame") return sizeof(cticp_synthetic_frame);
    if (s == "cticp_lidar_sensor") return sizeof(cticp_lidar_sensor);
    if (s == "cticp_lidar_frame") return sizeof(cticp_lidar_frame);
    if (s == "cticp_nclt_frame") return sizeof(cticp_nclt_frame);
    if (s == "cticp_ply_layout") return sizeof(cticp_ply_layout);
    if (s == "cticp_ply_property") return sizeof(cticp_ply_property);
    if (s == "cticp_strategy_options") return sizeof(cticp_strategy_options);
    if (s == "cticp_motion_model_options") return sizeof(cticp_motion_model_options);
    if (s == "cticp_odometry_options") return sizeof(cticp_odometry_options);
    if (s == "cticp_pose") return sizeof(cticp_pose);
    if (s == "cticp_frame") return sizeof(cticp_frame);
    if (s == "cticp_wpoint") return sizeof(cticp_wpoint);
    if (s == "cticp_icp_summary") return sizeof(cticp_icp_summary);
    if (s == "cticp_summary") return sizeof(cticp_summary);
    if (s == "cticp_device_timing") return sizeof(cticp_device_timing);
    if (s == "cticp_adaptive_options") return sizeof(cticp_adaptive_options);
    if (s == "cticp_device_scan") return sizeof(cticp_device_scan);
    if (s == "cticp_batch_frame") return sizeof(cticp_batch_frame);
    if (s == "cticp_kitti_errors") return sizeof(cticp_kitti_errors);
    if (s == "cticp_traj_segment") return sizeof(cticp_traj_segment);
    if (s == "cticp_traj_metrics") return sizeof(cticp_traj_metrics);
    return 0;
}

/* ---- defaults (include/ct_icp/ct_icp.h:60-152, map.h:115-125, odometry.h:37-157, motion_model.h:42-58) ------ */
void cticp_default_icp_options(cticp_icp_options *o) {
    memset(o, 0, sizeof(*o));
    o->num_iters_icp = 5;
    o->parametrization = CTICP_PARAM_CONTINUOUS_TIME;
    o->distance = CTICP_DIST_POINT_TO_PLANE;
    o->solver = CTICP_SOLVER_CERES;
    o->max_num_residuals = -1;
    o->min_num_residuals = 100;
    o->weighting_scheme = CTICP_WEIGHT_ALL;
    o->weight_alpha = 0.9;
    o->weight_neighborhood = 0.1;
    o->power_planarity = 2.0;
    o->max_number_neighbors = 20;
    o->min_number_neighbors = 20;
    o->threshold_voxel_occupancy = 1;
    o->num_closest_neighbors = 1;
    o->threshold_orientation_norm = 0.0001;
    o->threshold_translation_norm = 0.001;
    o->point_to_plane_with_distortion = 1;
    o->loss_function = CTICP_LOSS_CAUCHY;
    o->ls_max_num_iters = 1;
    o->ls_num_threads = 16;
    o->ls_sigma = 0.1;
    o->ls_tolerant_min_threshold = 0.05;
    o->max_dist_to_plane_ct_icp = 0.3;
    o->threshold_linearity = 0.8;
    o->threshold_planarity = 0.8;
    o->weight_point_to_point = 0.1;
    o->outlier_distance = 1.0;
    o->use_barycenter = 0;
    o->use_lines = 1;
    o->debug_print = 1;
}
void cticp_default_map_options(cticp_map_options *o) {
    memset(o, 0, sizeof(*o));
    o->num_resolutions = 3;
    o->resolutions[0].resolution = 0.2; o->resolutions[0].min_distance_between_points = 0.03; o->resolutions[0].max_num_points = 50;
    o->resolutions[1].resolution = 0.5; o->resolutions[1].min_distance_between_points = 0.1;  o->resolutions[1].max_num_points = 40;
    o->resolutions[2].resolution = 1.5; o->resolutions[2].min_distance_between_points = 0.15; o->resolutions[2].max_num_points = 40;
    o->select_valid_normals_direction = 1;
    o->max_frames_to_keep = 100;
    o->default_radius = 0.8;
}
void cticp_legacy_map_options(cticp_map_options *o, double size_voxel_map, int max_num_points_in_voxel,
                              double min_distance_points) {
    cticp_default_map_options(o);
    o->num_resolutions = 1;
    o->max_frames_to_keep = 1;
    o->resolutions[0].resolution = size_voxel_map;
    o->resolutions[0].max_num_points = max_num_points_in_voxel;
    o->resolutions[0].min_distance_between_points = min_distance_points;
}
void cticp_default_adaptive_options(cticp_adaptive_options *a) {   // include/ct_icp/algorithm/sampling.h:14-27
    memset(a, 0, sizeof(*a));
    a->num_points_per_voxel = 1;
    a->max_num_points = -1;
    a->num_bands = 6;
    const double d[6] = {0.5, 2.0, 4., 8., 16., 200.}, v[6] = {0.1, 0.2, 0.4, 0.8, 1.6, -1.};
    for (int i = 0; i < 6; ++i) {
        a->distance[i] = d[i];
        a->voxel_size[i] = v[i];
    }
}
void cticp_default_odometry_options(cticp_odometry_options *o) {
    memset(o, 0, sizeof(*o));
    cticp_default_adaptive_options(&o->adaptive_options);
    cticp_default_icp_options(&o->ct_icp_options);
    cticp_default_map_options(&o->map_options);
    o->neighborhood_strategy.type = 0;
    o->neighborhood_strategy.max_num_neighbors = 20;
    o->neighborhood_strategy.min_num_neighbors = 8;
    o->neighborhood_strategy.distance_max = 60.;   // DistanceBasedStrategy::Options, neighborhood_strategy.h:113-119
    o->neighborhood_strategy.radius_min = 0.1;
    o->neighborhood_strategy.radius_max = 2.0;
    o->neighborhood_strategy.exponent = 1.0;
    o->default_motion_model.model = CTICP_MM_CONSTANT_VELOCITY;
    o->default_motion_model.beta_location_consistency = 0.001;
    o->default_motion_model.beta_constant_velocity = 0.001;
    o->default_motion_model.beta_small_velocity = 0.0;
    o->default_motion_model.beta_orientation_consistency = 0.0;
    o->default_motion_model.threshold_orientation_deg = 15;
    o->default_motion_model.threshold_translation_diff = 0.3;
    o->default_motion_model.log_if_invalid = 1;
    o->motion_compensation = CTICP_MC_CONTINUOUS;
    o->initialization = CTICP_INIT_CONSTANT_VELOCITY;
    o->init_voxel_size = 0.2;
    o->init_sample_voxel_size = 1.0;
    o->init_num_frames = 20;
    o->sample_voxel_size = 1.5;
    o->max_num_keypoints = -1;
    o->sampling = CTICP_SAMPLING_GRID;
    o->voxel_size = 0.5;
    o->max_distance = 100.0;
    o->distance_error_threshold = 5.0;
    o->orientation_error_threshold = 30.;
    o->quit_on_error = 1;
    o->robust_minimal_level = 0;
    o->robust_registration = 0;
    o->robust_full_voxel_threshold = 0.7;
    o->robust_empty_voxel_threshold = 0.1;
    o->robust_neighborhood_min_dist = 0.10;
    o->robust_neighborhood_min_orientation = 0.1;
    o->robust_relative_trans_threshold = 1.0;
    o->robust_fail_early = 0;
    o->robust_num_attempts = 6;
    o->robust_num_attempts_when_rotation = 2;
    o->robust_max_voxel_neighborhood = 3;
    o->robust_threshold_ego_orientation = 3;
    o->robust_threshold_relative_orientation = 3;
    o->insertion_ego_rotation_threshold = 3;
    o->insertion_threshold_frames_skipped = 5;
    o->insertion_cum_distance_threshold = 0.8;
    o->insertion_cum_orientation_threshold = 5;
    o->always_insert = 0;
    o->do_no_insert = 0;
    o->debug_print = 1;
    o->with_default_motion_model = 1;
    o->shuffle_seed = 0x5DEECE66Dull;
    o->max_points_per_frame = 0;
}
void cticp_profile_default_driving(cticp_odometry_options *o) {
    cticp_default_odometry_options(o);
    o->ct_icp_options.solver = CTICP_SOLVER_CERES;
    o->ct_icp_options.ls_num_threads = 6;
    o->ct_icp_options.num_iters_icp = 5;
}
void cticp_profile_robust_driving(cticp_odometry_options *o) {
    cticp_default_odometry_options(o);
    o->voxel_size = 0.5;
    o->sample_voxel_size = 1.5;
    o->max_distance = 200.0;
    o->init_num_frames = 40;
    o->distance_error_threshold = 5.0;
    o->debug_print = 0;
    o->robust_registration = 1;
    o->robust_full_voxel_threshold = 0.5;
    o->robust_empty_voxel_threshold = 0.2;
    o->robust_num_attempts = 10;
    o->robust_max_voxel_neighborhood = 4;
    o->robust_threshold_relative_orientation = 5;
    o->robust_threshold_ego_orientation = 5;
    cticp_icp_options &c = o->ct_icp_options;
    c.debug_print = 0;
    c.max_number_neighbors = 20;
    c.min_number_neighbors = 20;
    c.num_iters_icp = 15;
    c.max_dist_to_plane_ct_icp = 0.5;
    c.threshold_orientation_norm = 0.01;
    c.num_closest_neighbors = 1;
    c.loss_function = CTICP_LOSS_CAUCHY;
    c.solver = CTICP_SOLVER_CERES;
    c.ls_max_num_iters = 20;
    c.ls_num_threads = 8;
    c.ls_sigma = 0.2;
    c.ls_tolerant_min_threshold = 0.05;
}
void cticp_profile_robust_outdoor_low_inertia(cticp_odometry_options *o) {
    cticp_default_odometry_options(o);
    o->voxel_size = 0.3;
    o->sample_voxel_size = 1.5;
    o->max_distance = 200.0;
    o->init_num_frames = 20;
    o->initialization = CTICP_INIT_NONE;
    o->debug_print = 0;
    o->robust_registration = 1;
    o->robust_full_voxel_threshold = 0.5;
    o->robust_empty_voxel_threshold = 0.1;
    o->robust_num_attempts = 3;
    o->robust_max_voxel_neighborhood = 4;
    o->robust_threshold_relative_orientation = 2;
    o->robust_threshold_ego_orientation = 2;
    o->default_motion_model.beta_constant_velocity = 0.0;
    o->default_motion_model.beta_location_consistency = 0.0;
    o->default_motion_model.beta_small_velocity = 0.001;
    o->default_motion_model.beta_orientation_consistency = 0.0;
    cticp_icp_options &c = o->ct_icp_options;
    c.num_iters_icp = 30;
    c.threshold_voxel_occupancy = 5;
    c.max_number_neighbors = 20;
    c.min_number_neighbors = 20;
    c.max_dist_to_plane_ct_icp = 0.5;
    c.threshold_orientation_norm = 0.01;
    c.num_closest_neighbors = 1;
    c.loss_function = CTICP_LOSS_CAUCHY;
    c.solver = CTICP_SOLVER_CERES;
    c.ls_max_num_iters = 10;
    c.ls_num_threads = 8;
    c.ls_sigma = 0.2;
    c.ls_tolerant_min_threshold = 0.05;
    c.weight_neighborhood = 0.2;
    c.weight_alpha = 0.8;
    c.weighting_scheme = CTICP_WEIGHT_ALL;
    c.max_num_residuals = 600;
    c.min_num_residuals = 200;
}

/* ---- Odometry ------------------------------------------------------------------------------------------------ */
int cticp_odometry_create(const cticp_odometry_options *options, int device, cticp_odometry **out) {
    return Guard([&] {
        if (!options || !out) throw std::invalid_argument("null argument");
        RequireDevice(device);
        auto h = std::make_unique<cticp_odometry>();
        h->engine = std::make_unique<Engine>(*options, device);
        h->map_view.map = &h->engine->Map();
        h->map_view.icp = &h->engine->Solver();
        h->map_view.stream = h->engine->Stream();
        h->map_view.device = device;
        h->map_view.owned = false;
        *out = h.release();
        return (int) CTICP_OK;
    });
}
void cticp_odometry_destroy(cticp_odometry *h) {
    delete h;
}
int cticp_odometry_register_frame(cticp_odometry *h, const double *xyz, size_t xyz_stride_bytes, const double *t,
                                  size_t t_stride_bytes, size_t n, uint32_t frame_id,
                                  const cticp_frame *initial_estimate, cticp_summary *out_summary) {
    return Guard([&] {
        if (!h) throw std::invalid_argument("null handle");
        cticp::ScanView v;
        v.xyz = xyz; v.xyz_stride = xyz_stride_bytes; v.t = t; v.t_stride = t_stride_bytes; v.n = n;
        h->engine->RegisterFrame(v, frame_id, initial_estimate, out_summary);
        return (int) CTICP_OK;
    });
}
int cticp_odometry_register_frame_ex(cticp_odometry *h, const double *xyz, size_t xyz_stride_bytes, const double *t,
                                     size_t t_stride_bytes, size_t n, uint32_t frame_id,
                                     const cticp_frame *initial_estimate, const cticp_motion_prior *motion_model,
                                     cticp_summary *out_summary) {
    return Guard([&] {
        if (!h) throw std::invalid_argument("null handle");
        cticp::ScanView v;
        v.xyz = xyz; v.xyz_stride = xyz_stride_bytes; v.t = t; v.t_stride = t_stride_bytes; v.n = n;
        h->engine->RegisterFrame(v, frame_id, initial_estimate, out_summary, motion_model);
        return (int) CTICP_OK;
    });
}
int cticp_odometry_set_callback(cticp_odometry *h, cticp_event_fn fn, void *user) {
    return Guard([&] {
        if (!h) throw std::invalid_argument("null handle");
        h->engine->SetCallback(fn, user);
        return (int) CTICP_OK;
    });
}
int cticp_odometry_reset_options(cticp_odometry *h, const cticp_odometry_options *options) {
    return Guard([&] {
        if (!h || !options) throw std::invalid_argument("null argument");
        const int device = h->engine->Device();
        auto fresh = std::make_unique<Engine>(*options, device);   // throws before the old engine is touched
        h->engine = std::move(fresh);
        h->map_view.map = &h->engine->Map();
        h->map_view.icp = &h->engine->Solver();
        h->map_view.stream = h->engine->Stream();
        return (int) CTICP_OK;
    });
}
static cticp::ScanView ViewOfCloud(const cticp_cloud_view *c) {
    if (!c || !c->data) throw std::invalid_argument("The registered frame cannot be empty");
    const size_t xs = c->xyz_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8;
    static const size_t kSize[9] = {0, 1, 1, 2, 2, 4, 4, 4, 8};
    if (c->t_dtype < 1 || c->t_dtype > 8) throw std::invalid_argument("unknown timestamp dtype");
    if ((size_t) c->xyz_offset + 3 * xs > c->point_step || (size_t) c->t_offset + kSize[c->t_dtype] > c->point_step)
        throw std::invalid_argument("cloud view: a field lies outside the record (point_step)");
    cticp::ScanView v;
    v.xyz = static_cast<const char *>(c->data) + c->xyz_offset;
    v.xyz_stride = c->point_step;
    v.xyz_dtype = c->xyz_dtype;
    v.t = static_cast<const char *>(c->data) + c->t_offset;
    v.t_stride = c->point_step;
    v.t_dtype = c->t_dtype;
    v.n = (size_t) c->num_points;
    return v;
}
int cticp_odometry_register_cloud(cticp_odometry *h, const cticp_cloud_view *cloud, uint32_t frame_id,
                                  const cticp_frame *initial_estimate, cticp_summary *out_summary) {
    return Guard([&] {
        if (!h) throw std::invalid_argument("null handle");
        h->engine->RegisterFrame(ViewOfCloud(cloud), frame_id, initial_estimate, out_summary);
        return (int) CTICP_OK;
    });
}
int64_t cticp_odometry_stage_cloud(cticp_odometry *h, const cticp_cloud_view *cloud) {
    int64_t slot = -1;
    int rc = Guard([&] {
        slot = h->engine->StageFrame(ViewOfCloud(cloud));
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : slot;
}
int64_t cticp_odometry_write_points(cticp_odometry *h, int which, const cticp_cloud_sink *sink) {
    int64_t count = 0;
    int rc = Guard([&] {
        if (!sink) throw std::invalid_argument("null sink");
        count = h->engine->WritePoints(which, *sink);
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : count;
}
int cticp_odometry_register_device(cticp_odometry *h, const cticp_device_scan *scan, void *stream, uint32_t frame_id,
                                   const cticp_frame *initial_estimate, const cticp_motion_prior *motion_model,
                                   cticp_summary *out_summary) {
    return Guard([&] {
        if (!h || !scan) throw std::invalid_argument("null argument");
        cticp::ScanView v;
        v.xyz = scan->xyz; v.xyz_stride = scan->xyz_stride_bytes; v.xyz_dtype = scan->xyz_dtype;
        v.t = scan->t; v.t_stride = scan->t_stride_bytes; v.t_dtype = scan->t_dtype;
        v.n = (size_t) scan->num_points;
        h->engine->RegisterDevice(v, static_cast<cudaStream_t>(stream), frame_id, initial_estimate, out_summary, motion_model);
        return (int) CTICP_OK;
    });
}
int64_t cticp_odometry_write_points_device(cticp_odometry *h, int which, const cticp_cloud_sink *sink, void *stream) {
    int64_t count = 0;
    int rc = Guard([&] {
        if (!h || !sink) throw std::invalid_argument("null argument");
        count = h->engine->WritePointsDevice(which, *sink, static_cast<cudaStream_t>(stream));
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : count;
}
int64_t cticp_odometry_get_points(cticp_odometry *h, int which, cticp_wpoint *dst, size_t cap) {
    int64_t count = 0;
    int rc = Guard([&] {
        count = h->engine->GetPoints(which, dst, cap);
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : count;
}
int cticp_odometry_set_summary_points(cticp_odometry *h, int mask) {
    return Guard([&] {
        h->engine->SetSummaryPoints(mask);
        return (int) CTICP_OK;
    });
}
int64_t cticp_odometry_trajectory(cticp_odometry *h, cticp_frame *dst, size_t cap) {
    const auto &tr = h->engine->Trajectory();
    const size_t m = std::min(cap, tr.size());
    for (size_t i = 0; i < m && dst; ++i) dst[i] = FrameToC(tr[i]);
    return (int64_t) tr.size();
}
int64_t cticp_odometry_map_size(cticp_odometry *h) {
    int64_t v = 0;
    int rc = Guard([&] {
        v = h->engine->MapSize();
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : v;
}
int64_t cticp_odometry_map_points(cticp_odometry *h, double *dst_xyz, size_t cap_points) {
    return cticp_map_export(&h->map_view, 0, dst_xyz, nullptr, cap_points);
}
int cticp_odometry_reset(cticp_odometry *h) {
    return Guard([&] {
        h->engine->Reset();
        return (int) CTICP_OK;
    });
}
cticp_map *cticp_odometry_map(cticp_odometry *h) { return h ? &h->map_view : nullptr; }

/* ---- snapshots (snapshot.cu, snapshot_format.h) ----------------------------------------------------------------------- */
static cticp_odometry *WrapEngine(std::unique_ptr<Engine> engine) {
    auto h = std::make_unique<cticp_odometry>();
    h->engine = std::move(engine);
    h->map_view.map = &h->engine->Map();
    h->map_view.icp = &h->engine->Solver();
    h->map_view.stream = h->engine->Stream();
    h->map_view.device = h->engine->Device();
    h->map_view.owned = false;
    return h.release();
}
int64_t cticp_odometry_save(cticp_odometry *h, void *dst, size_t cap_bytes) {
    int64_t n = 0;
    const int rc = Guard([&] {
        if (!h) throw std::invalid_argument("null handle");
        n = h->engine->Save(dst, cap_bytes);
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : n;
}
int cticp_odometry_load(const void *src, size_t n_bytes, const cticp_odometry_options *options, int device,
                        cticp_odometry **out) {
    return Guard([&] {
        if (!src || !out) throw std::invalid_argument("null argument");
        RequireDevice(device);
        *out = WrapEngine(Engine::Load(src, n_bytes, options, device));
        return (int) CTICP_OK;
    });
}
int cticp_odometry_clone(cticp_odometry *h, int device, cticp_odometry **out) {
    return Guard([&] {
        if (!h || !out) throw std::invalid_argument("null argument");
        RequireDevice(device);
        *out = WrapEngine(h->engine->Clone(device));
        return (int) CTICP_OK;
    });
}
int cticp_odometry_last_timing(cticp_odometry *h, cticp_device_timing *out) {
    return Guard([&] {
        *out = h->engine->LastTiming();
        return (int) CTICP_OK;
    });
}
int64_t cticp_odometry_stage_frame(cticp_odometry *h, const double *xyz, size_t xyz_stride_bytes, const double *t,
                                   size_t t_stride_bytes, size_t n) {
    int64_t slot = -1;
    int rc = Guard([&] {
        cticp::ScanView v;
        v.xyz = xyz; v.xyz_stride = xyz_stride_bytes; v.t = t; v.t_stride = t_stride_bytes; v.n = n;
        slot = h->engine->StageFrame(v);
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : slot;
}
int cticp_odometry_register_staged(cticp_odometry *h, int64_t slot, uint32_t frame_id, cticp_summary *out_summary) {
    return Guard([&] {
        h->engine->RegisterStaged(slot, frame_id, out_summary);
        return (int) CTICP_OK;
    });
}
int cticp_odometry_register_batch(cticp_batch_frame *items, size_t batch) {
    std::vector<BatchItem> work;
    int rc = Guard([&] {
        if (!items || batch < 1 || batch > 64) throw std::invalid_argument("batch must hold 1 to 64 items");
        for (size_t i = 0; i < batch; ++i) {
            const cticp_batch_frame &it = items[i];
            const std::string at = "batch item " + std::to_string(i) + ": ";
            if (!it.handle || !it.handle->engine || !it.out) throw std::invalid_argument(at + "null handle or summary");
            if (it.kind == CTICP_BATCH_HOST) {
                if (!it.xyz || !it.t) throw std::invalid_argument(at + "null scan pointer");
            } else if (it.kind == CTICP_BATCH_DEVICE) {
                if (!it.device_scan) throw std::invalid_argument(at + "null device scan");
            } else if (it.kind == CTICP_BATCH_STAGED) {
                if (it.initial_estimate || it.motion_model)
                    throw std::invalid_argument(at + "a staged slot takes no initial estimate and no motion model");
            } else
                throw std::invalid_argument(at + "unknown kind");
            for (size_t j = 0; j < i; ++j)
                if (items[j].handle == it.handle) throw std::invalid_argument(at + "the same handle twice");
            if (it.handle->engine->Device() != items[0].handle->engine->Device())
                throw std::invalid_argument(at + "handles on different devices");
        }
        for (size_t i = 0; i < batch; ++i)
            if (items[i].handle->engine->ShardingMode() != 0)
                throw UnsupportedError("batch item " + std::to_string(i) + ": a sharded handle cannot join a batch");
        work.resize(batch);
        for (size_t i = 0; i < batch; ++i) {
            const cticp_batch_frame &it = items[i];
            BatchItem &w = work[i];
            w.engine = it.handle->engine.get();
            w.kind = it.kind;
            if (it.kind == CTICP_BATCH_HOST) {
                w.scan.xyz = it.xyz; w.scan.xyz_stride = it.xyz_stride_bytes; w.scan.t = it.t; w.scan.t_stride = it.t_stride_bytes;
                w.scan.n = it.n;
            } else if (it.kind == CTICP_BATCH_DEVICE) {
                const cticp_device_scan *d = it.device_scan;
                w.scan.xyz = d->xyz; w.scan.xyz_stride = d->xyz_stride_bytes; w.scan.xyz_dtype = d->xyz_dtype;
                w.scan.t = d->t; w.scan.t_stride = d->t_stride_bytes; w.scan.t_dtype = d->t_dtype;
                w.scan.n = (size_t) d->num_points;
                w.producer = static_cast<cudaStream_t>(it.stream);
            }
            w.slot = it.staged_slot;
            w.frame_id = it.frame_id;
            w.initial_estimate = it.initial_estimate;
            w.motion_model = it.motion_model;
            w.out = it.out;
        }
        return (int) CTICP_OK;
    });
    if (rc < 0) return rc;
    RegisterBatch(work);
    // every item's status; the message of the first failing one is left in cticp_last_error (set last)
    int first = CTICP_OK;
    for (size_t i = batch; i-- > 0;) {
        items[i].status = CTICP_OK;
        if (work[i].error) {
            const std::exception_ptr e = work[i].error;
            items[i].status = Guard([&]() -> int { std::rethrow_exception(e); });
            first = items[i].status;
        }
    }
    return first;
}
int cticp_odometry_clear_staged(cticp_odometry *h) {
    return Guard([&] {
        h->engine->ClearStaged();
        return (int) CTICP_OK;
    });
}
int cticp_odometry_timer_start(cticp_odometry *h) {
    return Guard([&] {
        h->engine->TimerStart();
        return (int) CTICP_OK;
    });
}
int cticp_odometry_timer_stop(cticp_odometry *h, double *elapsed_ms) {
    return Guard([&] {
        *elapsed_ms = h->engine->TimerStop();
        return (int) CTICP_OK;
    });
}
int cticp_odometry_flush_l2(cticp_odometry *h, size_t bytes) {
    return Guard([&] {
        h->engine->FlushL2(bytes);
        return (int) CTICP_OK;
    });
}
int cticp_odometry_set_gather_timing(cticp_odometry *h, int on) {
    h->engine->SetTimeGather(on != 0);
    return CTICP_OK;
}
int cticp_odometry_enable_sharding(cticp_odometry *h, const void *unique_id_128_bytes, int rank, int world) {
    return Guard([&] {
        h->engine->EnableSharding(unique_id_128_bytes, rank, world);
        return (int) CTICP_OK;
    });
}
int cticp_odometry_sharding_mode(cticp_odometry *h) { return h->engine->ShardingMode(); }

/* ---- continuous trajectories (trajectory.cu) ------------------------------------------------------------------------ */
int cticp_trajectory_create(const cticp_pose *poses, size_t n, int device, cticp_trajectory **out) {
    return Guard([&] {
        if (!poses || !out) throw std::invalid_argument("null argument");
        RequireDevice(device);
        auto t = std::make_unique<cticp_trajectory>();
        t->impl = std::make_unique<ContinuousTrajectory>(poses, n, device);
        *out = t.release();
        return (int) CTICP_OK;
    });
}
void cticp_trajectory_destroy(cticp_trajectory *t) { delete t; }
int64_t cticp_trajectory_poses(cticp_trajectory *t, cticp_pose *dst, size_t cap) {
    if (!t) return Fail(CTICP_ERR_INVALID_ARGUMENT, "null handle");
    const auto &p = t->impl->Poses();
    const size_t m = std::min(cap, p.size());
    for (size_t i = 0; i < m && dst; ++i) dst[i] = p[i];
    return (int64_t) p.size();
}
int cticp_trajectory_interpolate(cticp_trajectory *t, const double *timestamps, const uint32_t *frame_ids, size_t m,
                                 cticp_pose *out) {
    return Guard([&] {
        if (!t) throw std::invalid_argument("null handle");
        t->impl->Interpolate(timestamps, frame_ids, m, out);
        return (int) CTICP_OK;
    });
}
int64_t cticp_trajectory_transform(cticp_trajectory *t, const cticp_cloud_view *cloud, const uint64_t *segment_ends,
                                   const uint32_t *segment_frame_ids, size_t num_segments, const cticp_cloud_sink *sink) {
    int64_t count = 0;
    int rc = Guard([&] {
        if (!t || !cloud || !sink) throw std::invalid_argument("null argument");
        count = t->impl->Transform(*cloud, segment_ends, segment_frame_ids, num_segments, *sink);
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : count;
}
int64_t cticp_trajectory_transform_device(cticp_trajectory *t, const cticp_device_scan *scan, const uint64_t *segment_ends,
                                          const uint32_t *segment_frame_ids, size_t num_segments,
                                          const cticp_cloud_sink *sink, void *stream) {
    int64_t count = 0;
    int rc = Guard([&] {
        if (!t || !scan || !sink) throw std::invalid_argument("null argument");
        count = t->impl->TransformDevice(*scan, segment_ends, segment_frame_ids, num_segments, *sink,
                                         static_cast<cudaStream_t>(stream));
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : count;
}

/* ---- world clouds (world_cloud.cu) ------------------------------------------------------------------------------ */
void cticp_default_grid_sampling_options(cticp_grid_sampling_options *out) {
    if (!out) return;
    *out = cticp_grid_sampling_options{};
    out->grid_size = 1.0;               // GridSamplingOptions, grid_sampling.h:12-16
    out->num_points_per_voxel = 1;
    out->max_num_points = -1;
}
int64_t cticp_sample_points_in_grid(int device, const cticp_grid_sampling_options *options, const double *xyz,
                                    size_t stride_bytes, size_t n, uint64_t *out_indices, size_t cap) {
    int64_t count = 0;
    int rc = Guard([&] {
        if (!options || (n && !xyz)) throw std::invalid_argument("null argument");
        WorldCloud::CheckOptions(*options);
        if (stride_bytes < 24 || stride_bytes > 0xFFFFFFFFull) throw std::invalid_argument("stride_bytes outside [24, 2^32)");
        RequireDevice(device);
        WorldCloud wc(*options, std::max<size_t>(n, 1), std::max<size_t>(n, 1), device);
        cticp_cloud_view v{};
        v.data = xyz;
        v.num_points = n;
        v.point_step = (uint32_t) stride_bytes;
        v.xyz_dtype = CTICP_DTYPE_FLOAT64;
        wc.Add(nullptr, v, nullptr, nullptr, 0, nullptr);
        cticp_cloud_sink sink{};
        sink.capacity_points = out_indices ? cap : 0;
        sink.world = 1;
        count = wc.Export(sink, out_indices);
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : count;
}
int cticp_world_cloud_create(const cticp_grid_sampling_options *options, uint64_t capacity_voxels,
                             uint64_t capacity_points, int device, cticp_world_cloud **out) {
    return Guard([&] {
        if (!options || !out) throw std::invalid_argument("null argument");
        WorldCloud::CheckOptions(*options);
        RequireDevice(device);
        auto wc = std::make_unique<cticp_world_cloud>();
        wc->impl = std::make_unique<WorldCloud>(*options, capacity_voxels, capacity_points, device);
        *out = wc.release();
        return (int) CTICP_OK;
    });
}
void cticp_world_cloud_destroy(cticp_world_cloud *wc) { delete wc; }
int cticp_world_cloud_add(cticp_world_cloud *wc, cticp_trajectory *trajectory, const cticp_cloud_view *cloud,
                          const uint64_t *segment_ends, const uint32_t *segment_frame_ids, size_t num_segments,
                          cticp_world_cloud_stats *stats_out) {
    return Guard([&] {
        if (!wc || !cloud) throw std::invalid_argument("null argument");
        wc->impl->Add(trajectory ? trajectory->impl.get() : nullptr, *cloud, segment_ends, segment_frame_ids,
                      num_segments, stats_out);
        return (int) CTICP_OK;
    });
}
int cticp_world_cloud_add_device(cticp_world_cloud *wc, cticp_trajectory *trajectory, const cticp_device_scan *scan,
                                 const uint64_t *segment_ends, const uint32_t *segment_frame_ids, size_t num_segments,
                                 cticp_world_cloud_stats *stats_out, void *stream) {
    return Guard([&] {
        if (!wc || !scan) throw std::invalid_argument("null argument");
        wc->impl->AddDevice(trajectory ? trajectory->impl.get() : nullptr, *scan, segment_ends, segment_frame_ids,
                            num_segments, stats_out, static_cast<cudaStream_t>(stream));
        return (int) CTICP_OK;
    });
}
int cticp_world_cloud_add_odometry(cticp_world_cloud *wc, cticp_odometry *odometry, cticp_world_cloud_stats *stats_out) {
    return Guard([&] {
        if (!wc || !odometry) throw std::invalid_argument("null argument");
        wc->impl->AddOdometry(*odometry->engine, stats_out);
        return (int) CTICP_OK;
    });
}
int64_t cticp_world_cloud_num_points(cticp_world_cloud *wc) {
    if (!wc) return Fail(CTICP_ERR_INVALID_ARGUMENT, "null handle");
    return (int64_t) wc->impl->NumPoints();
}
int64_t cticp_world_cloud_num_voxels(cticp_world_cloud *wc) {
    if (!wc) return Fail(CTICP_ERR_INVALID_ARGUMENT, "null handle");
    return (int64_t) wc->impl->NumVoxels();
}
int64_t cticp_world_cloud_export(cticp_world_cloud *wc, const cticp_cloud_sink *sink, uint64_t *src_index) {
    int64_t count = 0;
    int rc = Guard([&] {
        if (!wc || !sink) throw std::invalid_argument("null argument");
        count = wc->impl->Export(*sink, src_index);
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : count;
}
int64_t cticp_world_cloud_export_device(cticp_world_cloud *wc, const cticp_cloud_sink *sink, uint64_t *src_index,
                                        void *stream) {
    int64_t count = 0;
    int rc = Guard([&] {
        if (!wc || !sink) throw std::invalid_argument("null argument");
        count = wc->impl->ExportDevice(*sink, src_index, static_cast<cudaStream_t>(stream));
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : count;
}
int cticp_world_cloud_clear(cticp_world_cloud *wc) {
    return Guard([&] {
        if (!wc) throw std::invalid_argument("null handle");
        wc->impl->Clear();
        return (int) CTICP_OK;
    });
}

/* ---- synthetic scenes and sequences (synthetic.cu) -------------------------------------------------------------- */
int cticp_synthetic_scene_create(const double *triangles, size_t num_triangles, const double *lines, size_t num_lines,
                                 const double *spheres, size_t num_spheres, const double *balls, size_t num_balls,
                                 int device, cticp_synthetic_scene **out) {
    return Guard([&] {
        if (!out) throw std::invalid_argument("null argument");
        RequireDevice(device);
        auto sc = std::make_unique<cticp_synthetic_scene>();
        sc->impl = std::make_unique<SyntheticScene>(triangles, num_triangles, lines, num_lines, spheres, num_spheres, balls,
                                                    num_balls, device);
        *out = sc.release();
        return (int) CTICP_OK;
    });
}
void cticp_synthetic_scene_destroy(cticp_synthetic_scene *s) { delete s; }
int64_t cticp_synthetic_scene_num_primitives(cticp_synthetic_scene *s) {
    if (!s) return Fail(CTICP_ERR_INVALID_ARGUMENT, "null handle");
    return (int64_t) s->impl->NumPrimitives();
}
int cticp_synthetic_scene_distance(cticp_synthetic_scene *s, const double *points, size_t m, double *out) {
    return Guard([&] {
        if (!s || (m && (!points || !out))) throw std::invalid_argument("null argument");
        s->impl->Distance(points, m, out);
        return (int) CTICP_OK;
    });
}
int64_t cticp_synthetic_generate_points(cticp_synthetic_scene *s, size_t num_points_per_primitive, const double *location,
                                        double distance, uint64_t seed, double *xyz, size_t cap, uint32_t *src_index) {
    int64_t count = 0;
    int rc = Guard([&] {
        if (!s) throw std::invalid_argument("null handle");
        count = s->impl->GeneratePoints(num_points_per_primitive, location, distance, seed, xyz, cap, src_index);
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : count;
}
int64_t cticp_synthetic_generate_frames(cticp_synthetic_scene *s, cticp_trajectory *t, const cticp_synthetic_frame *frames,
                                        size_t m, size_t num_points_per_primitive, double distance, uint64_t seed,
                                        const cticp_cloud_sink *sink, uint32_t *src_index, uint64_t *frame_ends) {
    int64_t count = 0;
    int rc = Guard([&] {
        if (!s || !t || !sink) throw std::invalid_argument("null argument");
        count = s->impl->GenerateFrames(*t->impl, frames, m, num_points_per_primitive, distance, seed, *sink, src_index,
                                        frame_ends);
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : count;
}
int cticp_synthetic_generate_frames_device(cticp_synthetic_scene *s, cticp_trajectory *t,
                                           const cticp_synthetic_frame *frames, size_t m,
                                           size_t num_points_per_primitive, double distance, uint64_t seed,
                                           const cticp_cloud_sink *sink, uint32_t *src_index, uint64_t *frame_ends,
                                           void *stream) {
    return Guard([&] {
        if (!s || !t || !sink) throw std::invalid_argument("null argument");
        s->impl->GenerateFramesDevice(*t->impl, frames, m, num_points_per_primitive, distance, seed, *sink, src_index,
                                      frame_ends, static_cast<cudaStream_t>(stream));
        return (int) CTICP_OK;
    });
}
int64_t cticp_synthetic_generate_poses(cticp_trajectory *t, double frequency, cticp_pose *out, size_t cap) {
    int64_t count = 0;
    int rc = Guard([&] {
        if (!t) throw std::invalid_argument("null handle");
        count = GeneratePoses(*t->impl, frequency, out, cap);
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : count;
}
int cticp_apply_uniform_noise(cticp_pose *poses, size_t n, double scale_rot_deg, double scale_trans_m, uint64_t seed) {
    return Guard([&] {
        if (n && !poses) throw std::invalid_argument("null argument");
        ApplyUniformNoise(poses, n, scale_rot_deg, scale_trans_m, seed);
        return (int) CTICP_OK;
    });
}

/* ---- spinning-LiDAR sweeps (lidar_sim.cu) ---------------------------------------------------------------------- */
int cticp_lidar_scene_create(const double *boxes, size_t num_boxes, const double *cylinders, size_t num_cylinders,
                             int ground, int device, cticp_lidar_scene **out) {
    return Guard([&] {
        if (!out) throw std::invalid_argument("null argument");
        RequireDevice(device);
        auto sc = std::make_unique<cticp_lidar_scene>();
        sc->impl = std::make_unique<LidarScene>(boxes, num_boxes, cylinders, num_cylinders, ground != 0, device);
        *out = sc.release();
        return (int) CTICP_OK;
    });
}
void cticp_lidar_scene_destroy(cticp_lidar_scene *s) { delete s; }
int cticp_lidar_scene_raycast(cticp_lidar_scene *s, const double *origins, const double *directions, size_t n,
                              double max_range, uint64_t seed, double *out) {
    return Guard([&] {
        if (!s) throw std::invalid_argument("null handle");
        s->impl->Raycast(origins, directions, n, max_range, seed, out);
        return (int) CTICP_OK;
    });
}
int cticp_lidar_scene_raycast_device(cticp_lidar_scene *s, const double *origins, const double *directions, size_t n,
                                     double max_range, uint64_t seed, double *out, void *stream) {
    return Guard([&] {
        if (!s) throw std::invalid_argument("null handle");
        s->impl->RaycastDevice(origins, directions, n, max_range, seed, out, static_cast<cudaStream_t>(stream));
        return (int) CTICP_OK;
    });
}
int64_t cticp_lidar_generate_sweeps(cticp_lidar_scene *s, cticp_trajectory *t, const cticp_lidar_sensor *sensor,
                                    const cticp_lidar_frame *frames, size_t m, uint64_t seed,
                                    const cticp_cloud_sink *sink, uint32_t *ray_index, uint64_t *frame_ends) {
    int64_t count = 0;
    int rc = Guard([&] {
        if (!s || !t || !sensor || !sink) throw std::invalid_argument("null argument");
        count = s->impl->GenerateSweeps(*t->impl, *sensor, frames, m, seed, *sink, ray_index, frame_ends);
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : count;
}
int cticp_lidar_generate_sweeps_device(cticp_lidar_scene *s, cticp_trajectory *t, const cticp_lidar_sensor *sensor,
                                       const cticp_lidar_frame *frames, size_t m, uint64_t seed,
                                       const cticp_cloud_sink *sink, uint32_t *ray_index, uint64_t *frame_ends,
                                       void *stream) {
    return Guard([&] {
        if (!s || !t || !sensor || !sink) throw std::invalid_argument("null argument");
        s->impl->GenerateSweepsDevice(*t->impl, *sensor, frames, m, seed, *sink, ray_index, frame_ends,
                                      static_cast<cudaStream_t>(stream));
        return (int) CTICP_OK;
    });
}

/* ---- dataset sequences (dataset.cu) ---------------------------------------------------------------------------- */
static int NcltOpen(const void *bytes, size_t n_bytes, uint32_t num_aggregated, int final, int device, bool on_device,
                    void *stream, cticp_nclt **out) {
    return Guard([&] {
        if (!out) throw std::invalid_argument("null argument");
        RequireDeviceCheap(device);
        auto h = std::make_unique<cticp_nclt>();
        h->impl = std::make_unique<NcltHits>(bytes, n_bytes, num_aggregated, final != 0, device, on_device,
                                             static_cast<cudaStream_t>(stream));
        *out = h.release();
        return (int) CTICP_OK;
    });
}
int cticp_nclt_open(const void *bytes, size_t n_bytes, uint32_t num_aggregated, int final, int device, cticp_nclt **out) {
    return NcltOpen(bytes, n_bytes, num_aggregated, final, device, false, nullptr, out);
}
int cticp_nclt_open_device(const void *bytes, size_t n_bytes, uint32_t num_aggregated, int final, int device,
                           void *stream, cticp_nclt **out) {
    return NcltOpen(bytes, n_bytes, num_aggregated, final, device, true, stream, out);
}
void cticp_nclt_destroy(cticp_nclt *h) { delete h; }
int64_t cticp_nclt_num_frames(const cticp_nclt *h) {
    return h ? (int64_t) h->impl->NumFrames() : Fail(CTICP_ERR_INVALID_ARGUMENT, "null handle");
}
int64_t cticp_nclt_num_packets(const cticp_nclt *h) {
    return h ? (int64_t) h->impl->NumPackets() : Fail(CTICP_ERR_INVALID_ARGUMENT, "null handle");
}
int64_t cticp_nclt_num_hits(const cticp_nclt *h) {
    return h ? (int64_t) h->impl->NumHits() : Fail(CTICP_ERR_INVALID_ARGUMENT, "null handle");
}
int64_t cticp_nclt_bytes_used(const cticp_nclt *h) {
    return h ? (int64_t) h->impl->BytesUsed() : Fail(CTICP_ERR_INVALID_ARGUMENT, "null handle");
}
int cticp_nclt_index_walked(const cticp_nclt *h) {
    return h ? (h->impl->Walked() ? 1 : 0) : Fail(CTICP_ERR_INVALID_ARGUMENT, "null handle");
}
int cticp_nclt_frame_info(const cticp_nclt *h, size_t first, size_t m, cticp_nclt_frame *out) {
    return Guard([&] {
        if (!h) throw std::invalid_argument("null handle");
        h->impl->FrameInfo(first, m, out);
        return (int) CTICP_OK;
    });
}
int64_t cticp_nclt_read_frames(cticp_nclt *h, size_t first, size_t m, const cticp_cloud_sink *sink,
                               uint64_t *frame_ends) {
    int64_t count = 0;
    int rc = Guard([&] {
        if (!h || !sink) throw std::invalid_argument("null argument");
        count = h->impl->ReadFrames(first, m, *sink, frame_ends);
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : count;
}
int cticp_nclt_read_frames_device(cticp_nclt *h, size_t first, size_t m, const cticp_cloud_sink *sink,
                                  uint64_t *frame_ends, void *stream) {
    return Guard([&] {
        if (!h || !sink) throw std::invalid_argument("null argument");
        h->impl->ReadFramesDevice(first, m, *sink, frame_ends, static_cast<cudaStream_t>(stream));
        return (int) CTICP_OK;
    });
}
int cticp_ply_layout_parse(const void *bytes, size_t n, cticp_ply_layout *out) {
    return Guard([&] {
        PlyLayoutParse(static_cast<const char *>(bytes), n, out);
        return (int) CTICP_OK;
    });
}

/* ---- PLY files (ply.cu) ---------------------------------------------------------------------------------------- */
int64_t cticp_ply_write(int device, const cticp_ply_property *props, size_t n_props, uint64_t num_items, void *out,
                        uint64_t capacity) {
    int64_t size = 0;
    const int rc = Guard([&] {
        RequireDeviceCheap(device);
        size = (int64_t) PlyWrite(device, props, n_props, num_items, out, capacity);
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : size;
}
int cticp_ply_write_device(int device, const cticp_ply_property *props, size_t n_props, uint64_t num_items,
                           const uint64_t *file_ends, size_t m, void *out, uint64_t capacity, uint64_t *file_offsets,
                           void *stream) {
    return Guard([&] {
        RequireDeviceCheap(device);
        PlyWriteDevice(device, props, n_props, num_items, file_ends, m, out, capacity, file_offsets,
                       static_cast<cudaStream_t>(stream));
        return (int) CTICP_OK;
    });
}
int64_t cticp_ply_read_poses(const void *bytes, size_t n, cticp_pose *out, size_t cap) {
    int64_t count = 0;
    const int rc = Guard([&] {
        const std::vector<cticp_pose> poses = PlyReadPoses(static_cast<const char *>(bytes), n);
        if (cap && !out) throw std::invalid_argument("null argument");
        for (size_t i = 0; i < poses.size() && i < cap; ++i) out[i] = poses[i];
        count = (int64_t) poses.size();
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : count;
}
int cticp_kitti_frame_filter_device(int device, const cticp_device_scan *scan, const cticp_cloud_sink *sink,
                                    void *stream) {
    return Guard([&] {
        if (!scan || !sink) throw std::invalid_argument("null argument");
        RequireDeviceCheap(device);
        KittiFrameFilterDevice(device, *scan, *sink, static_cast<cudaStream_t>(stream));
        return (int) CTICP_OK;
    });
}
int cticp_kitti_frame_filter(int device, const cticp_cloud_view *cloud, const cticp_cloud_sink *sink) {
    return Guard([&] {
        if (!cloud || !sink) throw std::invalid_argument("null argument");
        RequireDeviceCheap(device);
        KittiFrameFilter(device, *cloud, *sink);
        return (int) CTICP_OK;
    });
}
int cticp_scan_time_ranges_device(int device, const cticp_device_scan *scan, const uint64_t *frame_ends, size_t m,
                                  double *out_minmax, void *stream) {
    return Guard([&] {
        if (!scan) throw std::invalid_argument("null argument");
        RequireDeviceCheap(device);
        ScanTimeRangesDevice(device, *scan, frame_ends, m, out_minmax, static_cast<cudaStream_t>(stream));
        return (int) CTICP_OK;
    });
}
int cticp_scan_time_ranges(int device, const cticp_cloud_view *cloud, const uint64_t *frame_ends, size_t m,
                           double *out_minmax) {
    return Guard([&] {
        if (!cloud) throw std::invalid_argument("null argument");
        RequireDeviceCheap(device);
        ScanTimeRanges(device, *cloud, frame_ends, m, out_minmax);
        return (int) CTICP_OK;
    });
}
int64_t cticp_ground_truth_parse(int dataset, int sequence_id, const char *text, size_t n, cticp_pose *out, size_t cap) {
    int64_t count = 0;
    int rc = Guard([&] {
        const std::vector<cticp_pose> poses = GroundTruthParse(dataset, sequence_id, text, n);
        if (cap && !out) throw std::invalid_argument("null out");
        std::copy(poses.begin(), poses.begin() + std::min(cap, poses.size()), out);
        count = (int64_t) poses.size();
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : count;
}

/* ---- neighbourhoods of a point cloud (neighborhood.cu) ---------------------------------------------------------- */
int cticp_neighborhood_describe_sets(int device, const double *xyz, size_t stride_bytes, size_t n,
                                     const uint64_t *segment_ends, size_t num_sets, int values,
                                     double linearity_threshold, double planarity_threshold,
                                     cticp_neighborhood_description *out) {
    return Guard([&] {
        if ((n && !xyz) || (num_sets && (!segment_ends || !out))) throw std::invalid_argument("null argument");
        RequireDevice(device);
        DescribePointSets(device, xyz, stride_bytes, n, segment_ends, num_sets, values, linearity_threshold,
                          planarity_threshold, out);
        return (int) CTICP_OK;
    });
}
int cticp_neighborhood_create(const double *xyz, size_t stride_bytes, size_t n, int device, cticp_neighborhood **out) {
    return Guard([&] {
        if (!out || (n && !xyz)) throw std::invalid_argument("null argument");
        RequireDevice(device);
        auto nb = std::make_unique<cticp_neighborhood>();
        nb->impl = std::make_unique<NeighborhoodIndex>(device);
        nb->impl->BuildHost(xyz, stride_bytes, n);
        *out = nb.release();
        return (int) CTICP_OK;
    });
}
int cticp_neighborhood_create_device(const cticp_device_scan *scan, void *stream, int device, cticp_neighborhood **out) {
    return Guard([&] {
        if (!out || !scan) throw std::invalid_argument("null argument");
        RequireDevice(device);
        auto nb = std::make_unique<cticp_neighborhood>();
        nb->impl = std::make_unique<NeighborhoodIndex>(device);
        nb->impl->BuildDevice(*scan, static_cast<cudaStream_t>(stream));
        *out = nb.release();
        return (int) CTICP_OK;
    });
}
int cticp_neighborhood_create_world_cloud(cticp_world_cloud *wc, cticp_neighborhood **out) {
    return Guard([&] {
        if (!out || !wc) throw std::invalid_argument("null argument");
        RequireDevice(wc->impl->Device());
        auto nb = std::make_unique<cticp_neighborhood>();
        nb->impl = std::make_unique<NeighborhoodIndex>(wc->impl->Device());
        nb->impl->BuildWorldCloud(*wc->impl);
        *out = nb.release();
        return (int) CTICP_OK;
    });
}
void cticp_neighborhood_destroy(cticp_neighborhood *nb) { delete nb; }
int64_t cticp_neighborhood_num_points(cticp_neighborhood *nb) {
    if (!nb) return Fail(CTICP_ERR_INVALID_ARGUMENT, "null handle");
    return (int64_t) nb->impl->NumPoints();
}
int64_t cticp_neighborhood_num_rejected(cticp_neighborhood *nb) {
    if (!nb) return Fail(CTICP_ERR_INVALID_ARGUMENT, "null handle");
    return (int64_t) nb->impl->NumRejected();
}
int cticp_neighborhood_search(cticp_neighborhood *nb, const double *queries, size_t m, int k, double max_radius,
                              uint64_t *indices, double *d2, int32_t *counts) {
    return Guard([&] {
        if (!nb) throw std::invalid_argument("null handle");
        nb->impl->Search(queries, m, k, max_radius, indices, d2, counts);
        return (int) CTICP_OK;
    });
}
int cticp_neighborhood_search_device(cticp_neighborhood *nb, const double *queries, size_t m, int k, double max_radius,
                                     uint64_t *indices, double *d2, int32_t *counts, void *stream) {
    return Guard([&] {
        if (!nb) throw std::invalid_argument("null handle");
        nb->impl->SearchDevice(queries, m, k, max_radius, indices, d2, counts, static_cast<cudaStream_t>(stream));
        return (int) CTICP_OK;
    });
}
int cticp_neighborhood_describe(cticp_neighborhood *nb, const double *queries, size_t m, int k, double max_radius,
                                int values, double linearity_threshold, double planarity_threshold,
                                cticp_neighborhood_description *out) {
    return Guard([&] {
        if (!nb) throw std::invalid_argument("null handle");
        nb->impl->Describe(queries, m, k, max_radius, values, linearity_threshold, planarity_threshold, out);
        return (int) CTICP_OK;
    });
}
int cticp_neighborhood_describe_device(cticp_neighborhood *nb, const double *queries, size_t m, int k,
                                       double max_radius, int values, double linearity_threshold,
                                       double planarity_threshold, cticp_neighborhood_description *out, void *stream) {
    return Guard([&] {
        if (!nb) throw std::invalid_argument("null handle");
        nb->impl->DescribeDevice(queries, m, k, max_radius, values, linearity_threshold, planarity_threshold, out,
                                 static_cast<cudaStream_t>(stream));
        return (int) CTICP_OK;
    });
}

/* ---- Scoring against ground truth ------------------------------------------------------------------------------ */
int64_t cticp_kitti_evaluate(int device, const cticp_pose *gt, size_t n, const cticp_pose *est, size_t num_estimates,
                             const double *lengths, size_t num_lengths, cticp_kitti_errors *out, double *tab_errors,
                             size_t cap) {
    int64_t count = 0;
    int rc = Guard([&] {
        CheckKittiArgs(gt, n, est, num_estimates, lengths, num_lengths, out);
        RequireDevice(device);
        count = KittiEvaluate(gt, n, est, num_estimates, lengths, num_lengths, out, tab_errors, cap);
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : count;
}
int64_t cticp_trajectory_kitti_evaluate(cticp_trajectory *t, const cticp_pose *gt, size_t n, const double *lengths,
                                        size_t num_lengths, cticp_kitti_errors *out, double *tab_errors, size_t cap) {
    int64_t count = 0;
    int rc = Guard([&] {
        if (!t) throw std::invalid_argument("null handle");
        CheckKittiTrajectoryArgs(gt, n, lengths, num_lengths, out);
        count = KittiEvaluateTrajectory(*t->impl, gt, n, lengths, num_lengths, out, tab_errors, cap);
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : count;
}
int64_t cticp_trajectory_metrics(int device, const cticp_pose *gt, size_t n, const cticp_pose *est,
                                 size_t num_estimates, double segment_length, cticp_traj_metrics *out,
                                 cticp_traj_segment *segments, size_t cap) {
    int64_t count = 0;
    int rc = Guard([&] {
        CheckMetricsArgs(gt, n, est, num_estimates, segment_length, out);
        RequireDevice(device);
        count = TrajectoryMetrics(gt, n, est, num_estimates, segment_length, out, segments, cap);
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : count;
}
int cticp_trajectory_distances(int device, const cticp_pose *gt, size_t n, int kind, double *out) {
    return Guard([&] {
        CheckDistancesArgs(gt, n, kind, out);
        RequireDevice(device);
        TrajectoryDistances(gt, n, kind, out);
        return (int) CTICP_OK;
    });
}

/* ---- Map ----------------------------------------------------------------------------------------------------- */
int cticp_map_create(const cticp_map_options *options, int device, cticp_map **out) {
    return Guard([&] {
        if (!options || !out) throw std::invalid_argument("null argument");
        RequireDevice(device);
        auto m = std::make_unique<cticp_map>();
        m->device = device;
        m->owned = true;
        m->owned_stream = cticp::Stream(cudaStreamNonBlocking);
        m->stream = m->owned_stream.get();
        m->owned_map = std::make_unique<DeviceMap>(*options, m->stream, options->select_valid_normals_direction != 0);
        m->map = m->owned_map.get();
        m->owned_icp = std::make_unique<IcpSolver>(m->stream);
        m->icp = m->owned_icp.get();
        CT_CUDA_CHECK(cudaStreamSynchronize(m->stream));
        *out = m.release();
        return (int) CTICP_OK;
    });
}
void cticp_map_destroy(cticp_map *m) {
    if (!m || !m->owned) return;
    cudaSetDevice(m->device);
    cudaStreamSynchronize(m->stream);
    delete m;   // the solver and the map go before the stream (reverse declaration order)
}
int cticp_map_insert(cticp_map *m, const double *xyz, size_t stride_bytes, size_t n) {
    return cticp_map_insert_from(m, xyz, stride_bytes, n, nullptr);
}
int cticp_map_insert_from(cticp_map *m, const double *xyz, size_t stride_bytes, size_t n, const double origin[3]) {
    return Guard([&] {
        CT_CUDA_CHECK(cudaSetDevice(m->device));
        m->map->InsertHost(xyz, stride_bytes, n, origin ? V3{origin[0], origin[1], origin[2]} : V3{0, 0, 0});
        m->map->SyncCounters();
        m->map->MaintainTables();
        return (int) CTICP_OK;
    });
}
int cticp_map_remove_far(cticp_map *m, const double location[3], double distance) {
    return Guard([&] {
        CT_CUDA_CHECK(cudaSetDevice(m->device));
        m->map->RemoveFar(V3{location[0], location[1], location[2]}, distance);
        m->map->SyncCounters();
        m->map->MaintainTables();
        return (int) CTICP_OK;
    });
}
int64_t cticp_map_num_points(cticp_map *m, int map_idx) {
    int64_t v = 0;
    int rc = Guard([&] {
        CT_CUDA_CHECK(cudaSetDevice(m->device));
        if (map_idx < 0 || map_idx >= m->map->NumLevels()) throw std::invalid_argument("map_idx");
        v = (int64_t) m->map->SyncCounters()[map_idx].num_points;
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : v;
}
int64_t cticp_map_num_voxels(cticp_map *m, int map_idx) {
    int64_t v = 0;
    int rc = Guard([&] {
        CT_CUDA_CHECK(cudaSetDevice(m->device));
        if (map_idx < 0 || map_idx >= m->map->NumLevels()) throw std::invalid_argument("map_idx");
        v = (int64_t) m->map->SyncCounters()[map_idx].num_voxels;
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : v;
}
int64_t cticp_map_export(cticp_map *m, int map_idx, double *dst_xyz, int32_t *dst_voxel, size_t cap_points) {
    int64_t v = 0;
    int rc = Guard([&] {
        CT_CUDA_CHECK(cudaSetDevice(m->device));
        if (map_idx < 0 || map_idx >= m->map->NumLevels()) throw std::invalid_argument("map_idx");
        std::vector<double> xyz;
        std::vector<int> vox;
        const size_t n = m->map->Export(map_idx, xyz, vox);
        const size_t k = std::min(cap_points, n);
        if (dst_xyz) memcpy(dst_xyz, xyz.data(), sizeof(double) * 3 * k);
        if (dst_voxel) memcpy(dst_voxel, vox.data(), sizeof(int32_t) * 3 * k);
        v = (int64_t) n;
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : v;
}
int cticp_map_compute_neighborhoods(cticp_map *m, const double *queries_xyz, size_t n, int max_num_neighbors,
                                    double *out_points, int32_t *out_counts) {
    return Guard([&] {
        CT_CUDA_CHECK(cudaSetDevice(m->device));
        if (n == 0) return (int) CTICP_OK;
        DeviceArray<double> d_q, d_out;
        DeviceArray<int> d_cnt;
        d_q.reserve(3 * n, m->stream);
        d_out.reserve(3 * n * max_num_neighbors, m->stream);
        d_cnt.reserve(n, m->stream);
        CT_CUDA_CHECK(cudaMemcpyAsync(d_q.data(), queries_xyz, sizeof(double) * 3 * n, cudaMemcpyHostToDevice, m->stream));
        CT_CUDA_CHECK(cudaMemsetAsync(d_out.data(), 0, sizeof(double) * 3 * n * max_num_neighbors, m->stream));
        m->icp->Neighborhoods(*m->map, d_q.data(), n, max_num_neighbors, d_out.data(), d_cnt.data());
        CT_CUDA_CHECK(cudaMemcpyAsync(out_points, d_out.data(), sizeof(double) * 3 * n * max_num_neighbors, cudaMemcpyDeviceToHost, m->stream));
        CT_CUDA_CHECK(cudaMemcpyAsync(out_counts, d_cnt.data(), sizeof(int) * n, cudaMemcpyDeviceToHost, m->stream));
        CT_CUDA_CHECK(cudaStreamSynchronize(m->stream));
        return (int) CTICP_OK;
    });
}
int cticp_map_radius_search(cticp_map *m, const double *queries_xyz, const double *radiuses, size_t n,
                            int max_num_neighbors, const double *sensor_location, double *out_points,
                            int32_t *out_counts) {
    return Guard([&] {
        CT_CUDA_CHECK(cudaSetDevice(m->device));
        if (n == 0) return (int) CTICP_OK;
        if (!queries_xyz || !radiuses || !out_points || !out_counts) throw std::invalid_argument("null argument");
        DeviceArray<double> d_q, d_r, d_out;
        DeviceArray<int> d_cnt;
        d_q.reserve(3 * n, m->stream);
        d_r.reserve(n, m->stream);
        d_out.reserve(3 * n * max_num_neighbors, m->stream);
        d_cnt.reserve(n, m->stream);
        CT_CUDA_CHECK(cudaMemcpyAsync(d_q.data(), queries_xyz, sizeof(double) * 3 * n, cudaMemcpyHostToDevice, m->stream));
        CT_CUDA_CHECK(cudaMemcpyAsync(d_r.data(), radiuses, sizeof(double) * n, cudaMemcpyHostToDevice, m->stream));
        CT_CUDA_CHECK(cudaMemsetAsync(d_out.data(), 0, sizeof(double) * 3 * n * max_num_neighbors, m->stream));
        m->icp->RadiusSearch(*m->map, d_q.data(), d_r.data(), n, max_num_neighbors, sensor_location, d_out.data(), d_cnt.data());
        CT_CUDA_CHECK(cudaMemcpyAsync(out_points, d_out.data(), sizeof(double) * 3 * n * max_num_neighbors, cudaMemcpyDeviceToHost, m->stream));
        CT_CUDA_CHECK(cudaMemcpyAsync(out_counts, d_cnt.data(), sizeof(int) * n, cudaMemcpyDeviceToHost, m->stream));
        CT_CUDA_CHECK(cudaStreamSynchronize(m->stream));
        return (int) CTICP_OK;
    });
}
int64_t cticp_map_save(cticp_map *m, void *dst, size_t cap_bytes) {
    int64_t n = 0;
    const int rc = Guard([&] {
        if (!m) throw std::invalid_argument("null handle");
        CT_CUDA_CHECK(cudaSetDevice(m->device));
        CT_CUDA_CHECK(cudaStreamSynchronize(m->stream));   // (an odometry's map: its frames' work is on this stream)
        n = SaveMap(*m->map, dst, cap_bytes);
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : n;
}
int cticp_map_load(const void *src, size_t n_bytes, int device, cticp_map **out) {
    return Guard([&] {
        if (!src || !out) throw std::invalid_argument("null argument");
        snap::Parsed p;
        ValidateMapSnapshot(src, n_bytes, &p);
        RequireDevice(device);
        auto m = std::make_unique<cticp_map>();
        m->device = device;
        m->owned = true;
        m->owned_stream = cticp::Stream(cudaStreamNonBlocking);
        m->stream = m->owned_stream.get();
        // (the normals the snapshot keeps: an odometry's map keeps them only for the distance-based strategy)
        m->owned_map = std::make_unique<DeviceMap>(p.map.options, m->stream, p.map.has_normals != 0);
        m->map = m->owned_map.get();
        m->owned_icp = std::make_unique<IcpSolver>(m->stream);
        m->icp = m->owned_icp.get();
        m->map->LoadSection(p);
        *out = m.release();
        return (int) CTICP_OK;
    });
}
int cticp_map_clear(cticp_map *m) {
    return Guard([&] {
        CT_CUDA_CHECK(cudaSetDevice(m->device));
        m->map->Clear();
        m->map->SyncCounters();
        return (int) CTICP_OK;
    });
}

/* ---- Registration -------------------------------------------------------------------------------------------- */
namespace {
// TPose::GetAlphaTimestamp (types.h:192-219)
double AlphaOf(double t, double bts, double ets) {
    const double mn = std::min(bts, ets), mx = std::max(bts, ets);
    if (mn > t || mx < t) return 0.0;
    if (mn == mx) return 1.0;
    return (t - mn) / (mx - mn);
}
struct DeviceKeypoints {
    DeviceArray<float4> d_kp;
    DeviceArray<float4> d_lo;   // residual plane (se3.cuh load_raw); has_lo: some coordinate is not float32-representable
    bool has_lo = false;
    DeviceArray<int> d_n;
    DeviceArray<IcpState> d_state;
    const float4 *lo() const { return has_lo ? d_lo.data() : nullptr; }
};
// keypoints → (fp32 raw xyz, alpha) in kp[0..n) and its residual plane in lo[0..n); returns whether some value is not
// float32-representable. Throws TimestampError for a timestamp outside the frame, before writing anything else.
bool PackKeypoints(const cticp_wpoint *keypoints, size_t n, const cticp_frame *frame, float4 *kp, float4 *lo) {
    const double bts = frame->begin_pose.dest_timestamp, ets = frame->end_pose.dest_timestamp;
    for (size_t i = 0; i < n; ++i) {
        const double t = keypoints[i].timestamp;
        if (!(bts <= t && t <= ets)) throw TimestampError("The timestamp cannot be interpolated between the two poses");
    }
    bool has_lo = false;
    for (size_t i = 0; i < n; ++i) {
        const double t = keypoints[i].timestamp;
        const double v[4] = {keypoints[i].raw[0], keypoints[i].raw[1], keypoints[i].raw[2], AlphaOf(t, bts, ets)};
        kp[i] = make_float4((float) v[0], (float) v[1], (float) v[2], (float) v[3]);
        lo[i] = make_float4((float) (v[0] - (double) kp[i].x), (float) (v[1] - (double) kp[i].y),
                            (float) (v[2] - (double) kp[i].z), (float) (v[3] - (double) kp[i].w));
        if (lo[i].x != 0.f || lo[i].y != 0.f || lo[i].z != 0.f || lo[i].w != 0.f) has_lo = true;
    }
    return has_lo;
}
// the registration state at the initial frame (+ PreviousFrameMotionModel when previous_frame and mo are given)
void InitialState(const cticp_frame *frame, const cticp_frame *previous_frame, const cticp_motion_model_options *mo,
                  IcpState &S);
void UploadRegistrationInputs(cticp_map *m, const cticp_wpoint *keypoints, size_t n, const cticp_frame *frame,
                              const cticp_frame *previous_frame, const cticp_motion_model_options *mo,
                              DeviceKeypoints &D, IcpState &S) {
    std::vector<float4> kp(n), lo(n);
    D.has_lo = PackKeypoints(keypoints, n, frame, kp.data(), lo.data());
    D.d_kp.reserve(std::max<size_t>(n, 1), m->stream);
    D.d_lo.reserve(std::max<size_t>(n, 1), m->stream);
    CT_CUDA_CHECK(cudaMemcpyAsync(D.d_lo.data(), lo.data(), sizeof(float4) * n, cudaMemcpyHostToDevice, m->stream));
    D.d_n.reserve(1, m->stream);
    D.d_state.reserve(1, m->stream);
    const int ni = (int) n;
    InitialState(frame, previous_frame, mo, S);
    CT_CUDA_CHECK(cudaMemcpyAsync(D.d_kp.data(), kp.data(), sizeof(float4) * n, cudaMemcpyHostToDevice, m->stream));
    CT_CUDA_CHECK(cudaMemcpyAsync(D.d_n.data(), &ni, sizeof(int), cudaMemcpyHostToDevice, m->stream));
    CT_CUDA_CHECK(cudaMemcpyAsync(D.d_state.data(), &S, sizeof(IcpState), cudaMemcpyHostToDevice, m->stream));
    CT_CUDA_CHECK(cudaStreamSynchronize(m->stream));
}
void InitialState(const cticp_frame *frame, const cticp_frame *previous_frame, const cticp_motion_model_options *mo,
                  IcpState &S) {
    memset(&S, 0, sizeof(S));
    const Q4 qb = qnormalized(Q4{frame->begin_pose.quat[0], frame->begin_pose.quat[1], frame->begin_pose.quat[2], frame->begin_pose.quat[3]});
    const Q4 qe = qnormalized(Q4{frame->end_pose.quat[0], frame->end_pose.quat[1], frame->end_pose.quat[2], frame->end_pose.quat[3]});
    S.qb[0] = qb.x; S.qb[1] = qb.y; S.qb[2] = qb.z; S.qb[3] = qb.w;
    S.qe[0] = qe.x; S.qe[1] = qe.y; S.qe[2] = qe.z; S.qe[3] = qe.w;
    for (int d = 0; d < 3; ++d) {
        S.tb[d] = frame->begin_pose.tr[d];
        S.te[d] = frame->end_pose.tr[d];
    }
    if (previous_frame && mo) {
        S.has_motion_model = 1;
        S.beta_location = mo->beta_location_consistency;
        S.beta_cv = mo->beta_constant_velocity;
        S.beta_small = mo->beta_small_velocity;
        S.beta_orientation = mo->beta_orientation_consistency;
        for (int d = 0; d < 3; ++d) {
            S.prev_tb[d] = previous_frame->begin_pose.tr[d];
            S.prev_te[d] = previous_frame->end_pose.tr[d];
        }
        for (int d = 0; d < 4; ++d) S.prev_qe[d] = previous_frame->end_pose.quat[d];
    }
    icp_state_refresh_slerp(S);
}
// The final state → the frame (in/out), the rewritten world points and the summary: what cticp_icp_register reports
void WriteRegistrationOutputs(const IcpState &S, cticp_wpoint *keypoints, size_t n, cticp_frame *frame,
                              cticp_icp_summary *out_summary) {
    for (int d = 0; d < 4; ++d) {
        frame->begin_pose.quat[d] = S.qb[d];
        frame->end_pose.quat[d] = S.qe[d];
    }
    for (int d = 0; d < 3; ++d) {
        frame->begin_pose.tr[d] = S.tb[d];
        frame->end_pose.tr[d] = S.te[d];
    }
    // world_kpts[i] ← InterpolatePose(begin, end, t_i) * raw_i with the final pose pair (ct_icp.cpp:964-966, :688)
    const Q4 qb{S.qb[0], S.qb[1], S.qb[2], S.qb[3]}, qe{S.qe[0], S.qe[1], S.qe[2], S.qe[3]};
    const V3 tb{S.tb[0], S.tb[1], S.tb[2]}, te{S.te[0], S.te[1], S.te[2]};
    const double bts = frame->begin_pose.dest_timestamp, ets = frame->end_pose.dest_timestamp;
    for (size_t i = 0; i < n; ++i) {
        const V3 w = ct_transform(qb, tb, qe, te, AlphaOf(keypoints[i].timestamp, bts, ets),
                                  V3{keypoints[i].raw[0], keypoints[i].raw[1], keypoints[i].raw[2]});
        keypoints[i].world[0] = w.x; keypoints[i].world[1] = w.y; keypoints[i].world[2] = w.z;
    }
    if (out_summary) {
        memset(out_summary, 0, sizeof(*out_summary));
        out_summary->success = !S.failed;
        out_summary->num_residuals_used = S.n_used;
        out_summary->num_iters = S.iter;
    }
}
}  // namespace

int cticp_icp_register(cticp_map *m, const cticp_icp_options *options, const cticp_strategy_options *strategy,
                       cticp_wpoint *keypoints, size_t n, cticp_frame *frame, const cticp_frame *previous_frame,
                       const cticp_motion_model_options *motion_options, cticp_icp_summary *out_summary) {
    return Guard([&] {
        if (!m || !options || !keypoints || !frame) throw std::invalid_argument("null argument");
        CT_CUDA_CHECK(cudaSetDevice(m->device));
        DeviceKeypoints D;
        IcpState S;
        UploadRegistrationInputs(m, keypoints, n, frame, previous_frame, motion_options, D, S);
        cticp_strategy_options st{0, 20, 8, 0, 60., 0.1, 2.0, 1.0};
        if (strategy) st = *strategy;
        m->icp->set_keypoints_lo(D.lo());
        switch (options->solver) {
            case CTICP_SOLVER_GN:
                m->icp->EnqueueGaussNewton(*m->map, *options, D.d_kp.data(), D.d_n.data(), n, options->num_iters_icp, D.d_state.data());
                break;
            case CTICP_SOLVER_CERES:
            case CTICP_SOLVER_ROBUST:
                m->icp->EnqueueCeres(*m->map, *options, st, D.d_kp.data(), D.d_n.data(), n, n, D.d_state.data());
                break;
            default:
                throw UnsupportedError("Unsupported Solver Type");
        }
        CT_CUDA_CHECK(cudaMemcpyAsync(&S, D.d_state.data(), sizeof(IcpState), cudaMemcpyDeviceToHost, m->stream));
        CT_CUDA_CHECK(cudaStreamSynchronize(m->stream));
        WriteRegistrationOutputs(S, keypoints, n, frame, out_summary);
        if (S.failed == 2) throw std::runtime_error("Error During Optimization");
        if (S.failed) g_last_error = "[CT_ICP]Error : not enough keypoints selected in ct-icp !";
        return (int) CTICP_OK;
    });
}

namespace {
// cticp_icp_register_batch(_ex): the problems' shared arguments are checked, then every problem's inputs (timestamps) are
// checked and packed before anything reaches the device; one batched launch of the solver's persistent kernel.
// gn_only: the entry without a strategy argument, which runs solver GN only.
int RegisterBatch(cticp_map *m, const cticp_icp_options *options, const cticp_strategy_options *strategy, size_t batch,
                  cticp_wpoint *const *keypoints, const size_t *n, cticp_frame *frames,
                  const cticp_frame *const *previous_frames, const cticp_motion_model_options *motion_options,
                  cticp_icp_summary *out_summaries, bool gn_only) {
    return Guard([&] {
        if (!m || !options || !keypoints || !n || !frames) throw std::invalid_argument("null argument");
        if (batch == 0 || batch > 64) throw std::invalid_argument("batch must be in [1, 64]");
        size_t total = 0;
        for (size_t b = 0; b < batch; ++b) {
            if (!keypoints[b] && n[b] > 0) throw std::invalid_argument("null keypoints");
            total += n[b];
        }
        if (total > (size_t) INT32_MAX) throw std::invalid_argument("too many keypoints in one batch");
        if (gn_only && options->solver != CTICP_SOLVER_GN) throw UnsupportedError("cticp_icp_register_batch: solver GN only");
        cticp_strategy_options st{0, 20, 8, 0, 60., 0.1, 2.0, 1.0};   // cticp_icp_register's default
        if (strategy) st = *strategy;
        const bool gn = options->solver == CTICP_SOLVER_GN;
        if (gn) {
            if (options->max_number_neighbors > 32 || options->max_number_neighbors < 1)
                throw UnsupportedError("max_number_neighbors must be in [1, 32]");
        } else if (options->solver != CTICP_SOLVER_CERES && options->solver != CTICP_SOLVER_ROBUST) {
            throw UnsupportedError("Unsupported Solver Type");
        }
        CT_CUDA_CHECK(cudaSetDevice(m->device));
        if (gn && !m->icp->batch_supported())
            throw UnsupportedError("cticp_icp_register_batch needs the persistent Gauss-Newton loop with flag synchronisation");
        if (!gn) {
            if (!m->icp->use_persistent())
                throw UnsupportedError("cticp_icp_register_batch_ex needs the persistent LM loop (CTICP_PERSISTENT)");
            m->icp->CheckCeresOptions(*m->map, *options, st);
        }
        // every problem's inputs are checked (timestamps) and packed before anything reaches the device
        std::vector<float4> kp(std::max<size_t>(total, 1)), lo(std::max<size_t>(total, 1));
        std::vector<IcpState> S(batch);
        std::vector<char> has_lo(batch);
        bool any_lo = false;
        for (size_t b = 0, base = 0; b < batch; base += n[b], ++b) {
            has_lo[b] = PackKeypoints(keypoints[b], n[b], &frames[b], kp.data() + base, lo.data() + base);
            any_lo = any_lo || has_lo[b];
            InitialState(&frames[b], previous_frames ? previous_frames[b] : nullptr, motion_options, S[b]);
        }
        if (any_lo)   // a problem that a solo call would run without a residual plane gets -0.0f: x + (-0.0) == x, every x
            for (size_t b = 0, base = 0; b < batch; base += n[b], ++b)
                if (!has_lo[b])
                    for (size_t i = 0; i < n[b]; ++i) lo[base + i] = make_float4(-0.f, -0.f, -0.f, -0.f);
        DeviceArray<float4> d_kp, d_lo;
        DeviceArray<IcpState> d_states;
        d_kp.reserve(kp.size(), m->stream);
        d_states.reserve(batch, m->stream);
        CT_CUDA_CHECK(cudaMemcpyAsync(d_kp.data(), kp.data(), sizeof(float4) * total, cudaMemcpyHostToDevice, m->stream));
        if (any_lo) {
            d_lo.reserve(lo.size(), m->stream);
            CT_CUDA_CHECK(cudaMemcpyAsync(d_lo.data(), lo.data(), sizeof(float4) * total, cudaMemcpyHostToDevice, m->stream));
        }
        CT_CUDA_CHECK(cudaMemcpyAsync(d_states.data(), S.data(), sizeof(IcpState) * batch, cudaMemcpyHostToDevice, m->stream));
        m->icp->set_keypoints_lo(d_lo.data());
        if (gn)
            m->icp->EnqueueGaussNewtonBatch(*m->map, *options, (int) batch, n, d_kp.data(), options->num_iters_icp, d_states.data());
        else
            m->icp->EnqueueCeresBatch(*m->map, *options, st, (int) batch, n, d_kp.data(), d_states.data());
        CT_CUDA_CHECK(cudaMemcpyAsync(S.data(), d_states.data(), sizeof(IcpState) * batch, cudaMemcpyDeviceToHost, m->stream));
        CT_CUDA_CHECK(cudaStreamSynchronize(m->stream));
        bool timeout = false, not_enough = false;
        for (size_t b = 0; b < batch; ++b) {
            WriteRegistrationOutputs(S[b], keypoints[b], n[b], &frames[b], out_summaries ? &out_summaries[b] : nullptr);
            timeout = timeout || S[b].failed == 2;
            not_enough = not_enough || S[b].failed;
        }
        if (timeout) throw std::runtime_error("Error During Optimization");
        if (not_enough) g_last_error = "[CT_ICP]Error : not enough keypoints selected in ct-icp !";
        return (int) CTICP_OK;
    });
}
}  // namespace

int cticp_icp_register_batch(cticp_map *m, const cticp_icp_options *options, size_t batch,
                             cticp_wpoint *const *keypoints, const size_t *n, cticp_frame *frames,
                             const cticp_frame *const *previous_frames, const cticp_motion_model_options *motion_options,
                             cticp_icp_summary *out_summaries) {
    return RegisterBatch(m, options, nullptr, batch, keypoints, n, frames, previous_frames, motion_options, out_summaries,
                         true);
}

int cticp_icp_register_batch_ex(cticp_map *m, const cticp_icp_options *options, const cticp_strategy_options *strategy,
                                size_t batch, cticp_wpoint *const *keypoints, const size_t *n, cticp_frame *frames,
                                const cticp_frame *const *previous_frames,
                                const cticp_motion_model_options *motion_options, cticp_icp_summary *out_summaries) {
    return RegisterBatch(m, options, strategy, batch, keypoints, n, frames, previous_frames, motion_options, out_summaries,
                         false);
}

int cticp_icp_gn_normal_equations(cticp_map *m, const cticp_icp_options *options, const cticp_wpoint *keypoints,
                                  size_t n, const cticp_frame *frame, const cticp_frame *previous_frame,
                                  const cticp_motion_model_options *motion_options, double *out_A144, double *out_b12,
                                  int32_t *out_num_used) {
    return Guard([&] {
        if (!m || !options || !keypoints || !frame) throw std::invalid_argument("null argument");
        CT_CUDA_CHECK(cudaSetDevice(m->device));
        DeviceKeypoints D;
        IcpState S;
        UploadRegistrationInputs(m, keypoints, n, frame, previous_frame, motion_options, D, S);
        int n_used = 0;
        m->icp->set_keypoints_lo(D.lo());
        m->icp->NormalEquations(*m->map, *options, D.d_kp.data(), D.d_n.data(), n, D.d_state.data(), out_A144, out_b12, &n_used);
        *out_num_used = n_used;
        return (int) CTICP_OK;
    });
}

/* ---- Sampling / order contract ------------------------------------------------------------------------------- */
int64_t cticp_grid_sample_indices(int device, const double *xyz, size_t stride_bytes, size_t n, double voxel_size,
                                  uint32_t *out_indices, size_t cap) {
    int64_t total = 0;
    int rc = Guard([&] {
        RequireDevice(device);
        if (n == 0) return (int) CTICP_OK;
        const cticp::Stream stream(cudaStreamNonBlocking);
        {
            FramePipeline pipe(n, stream.get());
            float4 *stage = pipe.Staging(), *stage_lo = pipe.StagingLo();
            for (size_t i = 0; i < n; ++i) {
                const double *p = reinterpret_cast<const double *>(reinterpret_cast<const char *>(xyz) + stride_bytes * i);
                stage[i] = make_float4((float) p[0], (float) p[1], (float) p[2], 0.f);
                stage_lo[i] = make_float4((float) (p[0] - (double) stage[i].x), (float) (p[1] - (double) stage[i].y),
                                          (float) (p[2] - (double) stage[i].z), 0.f);
            }
            pipe.Upload(n);
            pipe.UploadLo(n);
            pipe.GridSelect(pipe.d_raw(), pipe.d_raw_lo(), nullptr, pipe.d_count_n(), n, voxel_size, 0, 0, 0, 0, 0, 0, 0.f,
                            pipe.d_frame_mut(), pipe.d_frame_lo_mut(), pipe.d_frame_src_mut(), pipe.d_count_frame());
            pipe.QueueCountsReadback();
            CT_CUDA_CHECK(cudaStreamSynchronize(stream.get()));
            total = pipe.h_counts()[1];
            const size_t k = std::min<size_t>(cap, (size_t) total);
            CT_CUDA_CHECK(cudaMemcpy(out_indices, pipe.d_frame_src(), sizeof(uint32_t) * k, cudaMemcpyDeviceToHost));
        }
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : total;
}
int64_t cticp_adaptive_sample_indices(int device, const cticp_adaptive_options *options, const double *xyz,
                                      size_t stride_bytes, size_t n, uint32_t *out_indices, size_t cap) {
    int64_t total = 0;
    int rc = Guard([&] {
        RequireDevice(device);
        if (n == 0 || !options) return (int) CTICP_OK;
        const cticp::Stream stream(cudaStreamNonBlocking);
        {
            FramePipeline pipe(n, stream.get());
            float4 *stage = pipe.Staging(), *stage_lo = pipe.StagingLo();
            for (size_t i = 0; i < n; ++i) {
                const double *p = reinterpret_cast<const double *>(reinterpret_cast<const char *>(xyz) + stride_bytes * i);
                stage[i] = make_float4((float) p[0], (float) p[1], (float) p[2], 0.f);
                stage_lo[i] = make_float4((float) (p[0] - (double) stage[i].x), (float) (p[1] - (double) stage[i].y),
                                          (float) (p[2] - (double) stage[i].z), 0.f);
            }
            pipe.Upload(n);
            pipe.UploadLo(n);
            pipe.AdaptiveSelect(*options, pipe.d_raw(), pipe.d_raw_lo(), nullptr, pipe.d_count_n(), n, pipe.d_frame_mut(),
                                pipe.d_frame_lo_mut(), pipe.d_frame_src_mut(), pipe.d_count_frame());
            pipe.QueueCountsReadback();
            CT_CUDA_CHECK(cudaStreamSynchronize(stream.get()));
            total = pipe.h_counts()[1];
            const size_t k = std::min<size_t>(cap, (size_t) total);
            CT_CUDA_CHECK(cudaMemcpy(out_indices, pipe.d_frame_src(), sizeof(uint32_t) * k, cudaMemcpyDeviceToHost));
        }
        return (int) CTICP_OK;
    });
    return rc < 0 ? rc : total;
}
int cticp_permutation(uint64_t seed, uint64_t counter, uint32_t n, uint32_t *out_perm) {
    // pure integer bijection (same __host__ __device__ code the kernels run): no device needed
    const Perm p = perm_make(seed, counter, n ? n : 1);
    for (uint32_t i = 0; i < n; ++i) out_perm[i] = perm_apply(p, i);
    return CTICP_OK;
}

int cticp_nccl_unique_id(void *out_128_bytes);   // nccl_shard.cu

}  // extern "C"
