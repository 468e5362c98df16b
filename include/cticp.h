/*
 * cticp.h — C ABI of the H100-native CT-ICP registration engine.
 *
 * This is the drop-in boundary underneath the C++ facade `ct_icp::Odometry`
 * (ct_icp_b200/include/ct_icp/odometry.h). Plain pointers and sizes only; no
 * C++/torch/Eigen types. Every entry point names the reference interface it
 * replaces (paths relative to the upstream tree, jedeschaud/ct_icp @ d467813).
 *
 * Conventions
 *   - return value: CTICP_OK (0) or a negative cticp_status; the message of the
 *     last failure is available through cticp_last_error().
 *   - quaternions are stored (x, y, z, w) like Eigen::Quaterniond::coeffs().
 *   - one handle owns one CUDA device context + stream; a handle is NOT
 *     re-entrant (same rule as the reference: callers serialise, see
 *     ros/catkin_ws/ct_icp_odometry/src/ct_icp_odometry_node.cxx:67).
 *   - input clouds are borrowed for the duration of the call only.
 *   - there is NO CPU fallback: cticp_create fails with CTICP_ERR_NO_DEVICE
 *     when no sm_90 (H100) device is usable.
 *   - ingest precision: a scan is kept on the device as (x, y, z, alpha) in
 *     fp32 — what LiDAR drivers emit (KITTI .bin, PointCloud2 FLOAT32) — and all
 *     geometry is evaluated in fp64 from there. The reference reads the scan
 *     through double-converting views (src/ct_icp/odometry.cpp:335-336), so for
 *     FLOAT32 sources the two agree exactly. FLOAT64 coordinates that fp32
 *     cannot hold travel with a second fp32 plane of residuals (value - fp32(value);
 *     hi + lo reproduces the double to ~2^-48 relative), uploaded only for such
 *     scans: the samplers then see the same voxel for every point as the
 *     reference does and the sample sets are identical
 *     (tests/test_gpu_parity_r2.py::test_fp64_scan_coordinates_and_timestamps).
 *     With FLOAT32 coordinates and wider timestamps alpha is rounded to fp32
 *     (<= 6e-8 of the sweep: <= 1e-6 m at 15 m/s); the timestamps returned in
 *     cticp_wpoint records are rebuilt from alpha.
 *   - multi-GPU (cticp_odometry_enable_sharding): ONE driving thread per rank —
 *     every exchange is a device-side rendezvous that needs all ranks' kernels in
 *     flight at once, so one host thread driving two handles in turn deadlocks
 *     until the exchange times out (CTICP_PEER_TIMEOUT_MS, default 30 s).
 */
#ifndef CTICP_H
#define CTICP_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CTICP_ABI_VERSION 1
#define CTICP_MAX_RESOLUTIONS 8

typedef enum cticp_status {
    CTICP_OK = 0,
    CTICP_ERR_INVALID_ARGUMENT = -1,
    CTICP_ERR_NO_DEVICE = -2,
    CTICP_ERR_CUDA = -3,
    CTICP_ERR_CAPACITY = -4,      /* a device table / block pool is full */
    CTICP_ERR_TIMESTAMP = -5,     /* reference: CHECK in TPose::InterpolatePose, include/SlamCore/types.h:456 */
    CTICP_ERR_UNSUPPORTED = -6,   /* option combination outside the built hot path */
    CTICP_ERR_NCCL = -7,
    CTICP_ERR_INTERNAL = -8,
    CTICP_ERR_CALLBACK = -9       /* a registered callback returned 0 (reference: CHECK, src/ct_icp/odometry.cpp:748) */
} cticp_status;

/* ---- enums mirroring the reference (same numeric order) ------------------------------------------------ */
/* include/ct_icp/ct_icp.h:35-39 */
/* scalar types of interleaved point records = sensor_msgs/PointField datatype codes
 * (ros/roscore/src/pc2_conversion.cxx:6-27, slam::PROPERTY_TYPE) */
enum { CTICP_DTYPE_INT8 = 1, CTICP_DTYPE_UINT8 = 2, CTICP_DTYPE_INT16 = 3, CTICP_DTYPE_UINT16 = 4,
       CTICP_DTYPE_INT32 = 5, CTICP_DTYPE_UINT32 = 6, CTICP_DTYPE_FLOAT32 = 7, CTICP_DTYPE_FLOAT64 = 8 };
enum { CTICP_SOLVER_GN = 0, CTICP_SOLVER_CERES = 1, CTICP_SOLVER_ROBUST = 2 };
/* include/ct_icp/ct_icp.h:41-47 */
enum { CTICP_LOSS_STANDARD = 0, CTICP_LOSS_CAUCHY = 1, CTICP_LOSS_HUBER = 2, CTICP_LOSS_TOLERANT = 3,
       CTICP_LOSS_TRUNCATED = 4 };
/* include/ct_icp/ct_icp.h:49-53 */
enum { CTICP_WEIGHT_PLANARITY = 0, CTICP_WEIGHT_NEIGHBORHOOD = 1, CTICP_WEIGHT_ALL = 2 };
/* include/ct_icp/cost_functions.h:17-20 (POSE_PARAMETRIZATION) */
enum { CTICP_PARAM_SIMPLE = 0, CTICP_PARAM_CONTINUOUS_TIME = 1 };
/* include/ct_icp/cost_functions.h:22-27 (ICP_DISTANCE) */
enum { CTICP_DIST_POINT_TO_PLANE = 0, CTICP_DIST_POINT_TO_POINT = 1, CTICP_DIST_POINT_TO_LINE = 2,
       CTICP_DIST_POINT_TO_DISTRIBUTION = 3 };
/* include/ct_icp/odometry.h:16-21 (MOTION_COMPENSATION) */
enum { CTICP_MC_NONE = 0, CTICP_MC_CONSTANT_VELOCITY = 1, CTICP_MC_ITERATIVE = 2, CTICP_MC_CONTINUOUS = 3 };
/* include/ct_icp/odometry.h:23-26 (INITIALIZATION) */
enum { CTICP_INIT_NONE = 0, CTICP_INIT_CONSTANT_VELOCITY = 1 };
/* include/ct_icp/odometry.h:27-31 (sampling::SAMPLING_OPTION) */
enum { CTICP_SAMPLING_NONE = 0, CTICP_SAMPLING_GRID = 1, CTICP_SAMPLING_ADAPTIVE = 2 };
/* include/ct_icp/motion_model.h:36-39 */
enum { CTICP_MM_CONSTANT_VELOCITY = 0, CTICP_MM_SMALL_VELOCITY = 1 };

/* ---- option PODs ------------------------------------------------------------------------------------------ */

/* ct_icp::CTICPOptions, include/ct_icp/ct_icp.h:56-153 (defaults: cticp_default_icp_options) */
typedef struct cticp_icp_options {
    int32_t num_iters_icp;
    int32_t parametrization;
    int32_t distance;
    int32_t solver;
    int32_t max_num_residuals;
    int32_t min_num_residuals;
    int32_t weighting_scheme;
    int32_t max_number_neighbors;
    int32_t min_number_neighbors;
    int32_t threshold_voxel_occupancy;
    int32_t num_closest_neighbors;
    int32_t point_to_plane_with_distortion;
    int32_t loss_function;
    int32_t ls_max_num_iters;
    int32_t ls_num_threads;
    int32_t debug_print;
    double weight_alpha;
    double weight_neighborhood;
    double power_planarity;
    double threshold_orientation_norm;
    double threshold_translation_norm;
    double ls_sigma;
    double ls_tolerant_min_threshold;
    double max_dist_to_plane_ct_icp;
    /* ROBUST solver params (include/ct_icp/ct_icp.h:133-141) */
    double threshold_linearity;
    double threshold_planarity;
    double weight_point_to_point;
    double outlier_distance;
    int32_t use_barycenter;
    int32_t use_lines;             /* ct_icp.h:140 (default true; not settable from the reference's YAML) */
} cticp_icp_options;

/* ct_icp::MultipleResolutionVoxelMap::ResolutionParam / Options, include/ct_icp/map.h:109-134 */
typedef struct cticp_resolution_param {
    double resolution;
    double min_distance_between_points;
    int32_t max_num_points;
    int32_t _pad0;
} cticp_resolution_param;

typedef struct cticp_map_options {
    int32_t num_resolutions;
    int32_t select_valid_normals_direction;
    int32_t max_frames_to_keep;
    int32_t _pad0;
    double default_radius;
    cticp_resolution_param resolutions[CTICP_MAX_RESOLUTIONS];
    /* device sizing (new; not in the reference): 0 = pick from defaults */
    uint64_t capacity_voxels;      /* slots per resolution (power of two is taken) */
} cticp_map_options;

/* ct_icp::INeighborStrategyOptions + DefaultNearestNeighborStrategy::Options + DistanceBasedStrategy::Options,
 * include/ct_icp/neighborhood_strategy.h:37-55, 60-85, 95-146. The strategy is consulted by solver CERES only
 * (src/ct_icp/ct_icp.cpp:571); GN and ROBUST search with the map's default radius. */
enum { CTICP_STRATEGY_NEAREST_NEIGHBOR = 0, CTICP_STRATEGY_DISTANCE_BASED = 1 };
typedef struct cticp_strategy_options {
    int32_t type;                  /* CTICP_STRATEGY_* */
    int32_t max_num_neighbors;
    int32_t min_num_neighbors;
    int32_t _pad0;
    /* DISTANCE_BASED_STRATEGY (:113-119): search radius grows with the keypoint's range; the map's per-point
     * normals reject neighbors whose surface faces away from the sensor (map.h:482-490) */
    double distance_max;
    double radius_min;
    double radius_max;
    double exponent;
} cticp_strategy_options;

/* ct_icp::PreviousFrameMotionModel::Options, include/ct_icp/motion_model.h:42-58 */
typedef struct cticp_motion_model_options {
    int32_t model;
    int32_t log_if_invalid;
    double beta_location_consistency;
    double beta_constant_velocity;
    double beta_small_velocity;
    double beta_orientation_consistency;
    double threshold_orientation_deg;
    double threshold_translation_diff;
} cticp_motion_model_options;

/* ct_icp::AdaptiveGridSamplingOptions, include/ct_icp/algorithm/sampling.h:14-27 */
#define CTICP_MAX_ADAPTIVE_BANDS 8
typedef struct cticp_adaptive_options {
    int32_t num_points_per_voxel;      /* only 1 is built */
    int32_t max_num_points;
    int32_t num_bands;                 /* entries of distance_voxel_size */
    int32_t _pad0;
    double distance[CTICP_MAX_ADAPTIVE_BANDS];     /* .first  : distance to the sensor */
    double voxel_size[CTICP_MAX_ADAPTIVE_BANDS];   /* .second : sampling voxel of the band starting there */
} cticp_adaptive_options;

/* ct_icp::OdometryOptions, include/ct_icp/odometry.h:32-157 */
typedef struct cticp_odometry_options {
    cticp_icp_options ct_icp_options;
    cticp_map_options map_options;
    cticp_strategy_options neighborhood_strategy;
    cticp_motion_model_options default_motion_model;
    int32_t motion_compensation;
    int32_t initialization;
    int32_t init_num_frames;
    int32_t max_num_keypoints;
    int32_t sampling;
    int32_t quit_on_error;
    int32_t robust_minimal_level;
    int32_t robust_registration;
    int32_t robust_fail_early;
    int32_t robust_num_attempts;
    int32_t robust_num_attempts_when_rotation;
    int32_t robust_max_voxel_neighborhood;
    int32_t always_insert;
    int32_t do_no_insert;
    int32_t debug_print;
    int32_t with_default_motion_model;
    double init_voxel_size;
    double init_sample_voxel_size;
    double sample_voxel_size;
    double voxel_size;
    double max_distance;
    double distance_error_threshold;
    double orientation_error_threshold;
    double robust_full_voxel_threshold;
    double robust_empty_voxel_threshold;
    double robust_neighborhood_min_dist;
    double robust_neighborhood_min_orientation;
    double robust_relative_trans_threshold;
    double robust_threshold_ego_orientation;
    double robust_threshold_relative_orientation;
    double insertion_ego_rotation_threshold;
    double insertion_threshold_frames_skipped;
    double insertion_cum_distance_threshold;
    double insertion_cum_orientation_threshold;
    /* order contract (new): seed of the counter-based permutations that stand in for
     * std::shuffle(…, std::mt19937_64 g_) at src/ct_icp/odometry.cpp:349,361,550 */
    uint64_t shuffle_seed;
    /* device sizing (new): upper bound on points per scan; 0 = 524288 */
    uint64_t max_points_per_frame;
    cticp_adaptive_options adaptive_options;   /* sampling == ADAPTIVE */
} cticp_odometry_options;

/* ---- value PODs ------------------------------------------------------------------------------------------- */

/* slam::TPose<double>, include/SlamCore/types.h:162-274 */
typedef struct cticp_pose {
    double quat[4];                /* x, y, z, w */
    double tr[3];
    double ref_timestamp;
    double dest_timestamp;
    uint32_t ref_frame_id;
    uint32_t dest_frame_id;
} cticp_pose;

/* ct_icp::TrajectoryFrame, include/ct_icp/types.h:31-61 */
typedef struct cticp_frame {
    cticp_pose begin_pose;
    cticp_pose end_pose;
} cticp_frame;

/* slam::WPoint3D, include/SlamCore/types.h:35-60 (same 64-byte layout: raw xyz, t, world xyz, index_frame) */
typedef struct cticp_wpoint {
    double raw[3];
    double timestamp;
    double world[3];
    uint32_t index_frame;
    uint32_t _pad0;
} cticp_wpoint;

/* ct_icp::ICPSummary, include/ct_icp/ct_icp.h:155-169 */
typedef struct cticp_icp_summary {
    int32_t success;
    int32_t num_residuals_used;
    int32_t num_iters;
    int32_t _pad0;
    double duration_total;
    double duration_init;
    double avg_duration_iter;
    double avg_duration_neighborhood;
    double avg_duration_solve;
} cticp_icp_summary;

/* ct_icp::Odometry::RegistrationSummary, include/ct_icp/odometry.h:163-199.
 * The three point vectors are fetched on demand with cticp_odometry_get_points. */
typedef struct cticp_summary {
    cticp_frame frame;
    cticp_frame initial_frame;
    cticp_icp_summary icp_summary;
    int32_t sample_size;
    int32_t number_of_residuals;
    int32_t robust_level;
    int32_t success;
    int32_t points_added;
    int32_t number_of_attempts;
    double distance_correction;
    double relative_distance;
    double relative_orientation;
    double ego_orientation;
    uint64_t num_corrected_points;       /* F: points of the sub-sampled frame */
    uint64_t num_all_corrected_points;   /* N: points of the input scan */
    uint64_t num_keypoints;              /* K */
    /* logged_values (src/ct_icp/odometry.cpp:495-513), milliseconds */
    double odometry_total;
    double odometry_initialization;
    double odometry_try_register;
    double odometry_duration_sampling;
    double odometry_map_update;
    double odometry_transform;
    char error_message[256];
} cticp_summary;

enum { CTICP_POINTS_CORRECTED = 0, CTICP_POINTS_ALL_CORRECTED = 1, CTICP_POINTS_KEYPOINTS = 2 };

typedef struct cticp_odometry cticp_odometry;   /* opaque: replaces ct_icp::Odometry */
typedef struct cticp_map cticp_map;             /* opaque: replaces ct_icp::MultipleResolutionVoxelMap */

/* ---- defaults & profiles ---------------------------------------------------------------------------------- */
uint32_t cticp_abi_version(void);
const char *cticp_last_error(void);                                   /* thread-local */

void cticp_default_icp_options(cticp_icp_options *out);               /* include/ct_icp/ct_icp.h:60-152 */
void cticp_default_map_options(cticp_map_options *out);               /* include/ct_icp/map.h:115-125 */
void cticp_default_odometry_options(cticp_odometry_options *out);     /* include/ct_icp/odometry.h:37-157 */
void cticp_legacy_map_options(cticp_map_options *out, double size_voxel_map, int max_num_points_in_voxel,
                              double min_distance_points);            /* src/ct_icp/map.cpp:13-29 */
void cticp_profile_default_driving(cticp_odometry_options *out);      /* src/ct_icp/odometry.cpp:30-36 */
void cticp_profile_robust_driving(cticp_odometry_options *out);       /* src/ct_icp/odometry.cpp:39-89 */
void cticp_profile_robust_outdoor_low_inertia(cticp_odometry_options *out); /* src/ct_icp/odometry.cpp:92-151 */

/* ---- Odometry (L4 boundary) ------------------------------------------------------------------------------- */

/* ct_icp::Odometry::Odometry(const OdometryOptions&), src/ct_icp/odometry.cpp:697-734 */
int cticp_odometry_create(const cticp_odometry_options *options, int device, cticp_odometry **out);
void cticp_odometry_destroy(cticp_odometry *h);

/* ct_icp::Odometry::RegisterFrame(const slam::PointCloud&, frame_id_t, AMotionModel*), src/ct_icp/odometry.cpp:199-214
 * and RegisterFrameWithEstimate (:217-236) when initial_estimate != NULL.
 * xyz / t are strided HOST arrays (stride in bytes), the layout RegisterFrame reads through
 * XYZConst<double>() / TimestampsProxy<double>() (src/ct_icp/odometry.cpp:335-336). */
int cticp_odometry_register_frame(cticp_odometry *h,
                                  const double *xyz, size_t xyz_stride_bytes,
                                  const double *t, size_t t_stride_bytes,
                                  size_t n, uint32_t frame_id,
                                  const cticp_frame *initial_estimate,
                                  cticp_summary *out_summary);

/* The AMotionModel* argument of the RegisterFrame overloads (include/ct_icp/odometry.h:231-248). The reference's only
 * concrete model is PreviousFrameMotionModel (include/ct_icp/motion_model.h:35-78): its options and the previous frame it
 * was updated with. NULL = the reference's nullptr (the odometry's own default model when with_default_motion_model). */
typedef struct cticp_motion_prior {
    cticp_motion_model_options options;
    cticp_frame previous_frame;
} cticp_motion_prior;
int cticp_odometry_register_frame_ex(cticp_odometry *h,
                                     const double *xyz, size_t xyz_stride_bytes,
                                     const double *t, size_t t_stride_bytes,
                                     size_t n, uint32_t frame_id,
                                     const cticp_frame *initial_estimate,      /* nullable */
                                     const cticp_motion_prior *motion_model,   /* nullable */
                                     cticp_summary *out_summary);

/* ct_icp::Odometry::RegisterCallback (include/ct_icp/odometry.h:260, src/ct_icp/odometry.cpp:737-750): ONE hook per
 * handle, called on the registering thread at the reference's three events; inside it the caller may use
 * cticp_odometry_get_points (frame / keypoints with the pose pair of that moment). Returning 0 aborts the
 * registration with CTICP_ERR_CALLBACK. fn == NULL removes the hook. */
enum { CTICP_EVENT_BEFORE_ITERATION = 0, CTICP_EVENT_ITERATION_COMPLETED = 1, CTICP_EVENT_FINISHED_REGISTRATION = 2 };
typedef int (*cticp_event_fn)(int event, void *user);
int cticp_odometry_set_callback(cticp_odometry *h, cticp_event_fn fn, void *user);

/* An interleaved point buffer described like a sensor_msgs/PointCloud2 (one record every point_step bytes; field
 * "x" at xyz_offset with y and z following contiguously in the same scalar type — the "vertex" element that
 * SchemaBuilderFromCloud2 builds, ros/roscore/src/pc2_conversion.cxx:73-80 — and one timestamp scalar at t_offset).
 * It is the zero-copy input of the ROS node (ROSCloud2ToSlamPointCloudShallow, pc2_conversion.cxx:86-96 →
 * RegisterFrame(const slam::PointCloud&), src/ct_icp/odometry.cpp:199-214): the engine reads the records in place
 * and converts each scalar with static_cast<double>, as the reference's proxy views do
 * (include/SlamCore/data/view.h:99-120). Records need no alignment. */
typedef struct cticp_cloud_view {
    const void *data;
    uint64_t num_points;           /* width * height */
    uint32_t point_step;
    uint32_t xyz_offset;
    int32_t xyz_dtype;             /* CTICP_DTYPE_FLOAT32 or CTICP_DTYPE_FLOAT64 */
    uint32_t t_offset;
    int32_t t_dtype;               /* any CTICP_DTYPE_* */
    int32_t _pad0;
} cticp_cloud_view;

/* RegisterFrame(const slam::PointCloud&, frame_id) / RegisterFrameWithEstimate on a record buffer. */
int cticp_odometry_register_cloud(cticp_odometry *h, const cticp_cloud_view *cloud, uint32_t frame_id,
                                  const cticp_frame *initial_estimate, cticp_summary *out_summary);
/* cticp_odometry_stage_frame on a record buffer. */
int64_t cticp_odometry_stage_cloud(cticp_odometry *h, const cticp_cloud_view *cloud);

/* Egress in the caller's record layout (what the ROS node builds from summary.corrected_points / keypoints for its
 * publishers: pcl::PointCloud<slam::XYZTPoint>, ct_icp_odometry_node.cxx:228-262): writes world (world != 0) or raw
 * x,y,z and, when t_dtype != 0, the timestamp of min(capacity_points, count) points. Returns the count. */
typedef struct cticp_cloud_sink {
    void *data;
    uint64_t capacity_points;
    uint32_t point_step;
    uint32_t xyz_offset;
    int32_t xyz_dtype;             /* CTICP_DTYPE_FLOAT32 or CTICP_DTYPE_FLOAT64 */
    uint32_t t_offset;
    int32_t t_dtype;               /* 0 = no timestamp; else CTICP_DTYPE_FLOAT32 / CTICP_DTYPE_FLOAT64 */
    int32_t world;
} cticp_cloud_sink;
int64_t cticp_odometry_write_points(cticp_odometry *h, int which, const cticp_cloud_sink *sink);

/* RegistrationSummary::{corrected_points, all_corrected_points, keypoints}, include/ct_icp/odometry.h:187-191.
 * Copies min(cap, count) points device->host; returns the count or a negative status. */
int64_t cticp_odometry_get_points(cticp_odometry *h, int which, cticp_wpoint *dst, size_t cap);
/* RegistrationSummary returns its three point vectors BY VALUE from every RegisterFrame (src/ct_icp/odometry.cpp:462-486,
 * 597). mask: bit CTICP_POINTS_* set = that vector is produced eagerly by every following cticp_odometry_register_* call
 * (world coordinates transformed and copied to pinned host memory on a second stream, next to the map update), so the
 * cticp_odometry_get_points that follows only assembles the 64-byte records. 0 (default) = on demand. */
int cticp_odometry_set_summary_points(cticp_odometry *h, int mask);

/* Device input and output (new). A scan in device memory of the handle's device (cudaMalloc, cudaMallocManaged, a torch
 * CUDA tensor): x, y, z contiguous of one scalar type at xyz and one timestamp scalar at t, each strided in bytes. Records
 * need no alignment (PointCloud2 layouts: xyz = data + x_offset, t = data + t_offset, both strides = point_step). */
typedef struct cticp_device_scan {
    const void *xyz;
    uint64_t xyz_stride_bytes;
    const void *t;
    uint64_t t_stride_bytes;
    uint64_t num_points;
    int32_t xyz_dtype;             /* CTICP_DTYPE_FLOAT32 or CTICP_DTYPE_FLOAT64 */
    int32_t t_dtype;               /* any CTICP_DTYPE_* */
} cticp_device_scan;
/* cticp_odometry_register_frame_ex on a device scan: the same results, byte for byte, as on a host copy of the same values
 * and scalar types. The scan is packed on the device (no host round trip for the points). stream (a cudaStream_t; NULL =
 * the legacy default stream) is the producer's stream: the engine waits for its work through an event before reading. The
 * buffers may be overwritten once the call returns. Checked before anything is enqueued: pointers that are not device
 * memory of the handle's device, or a described buffer that extends past its allocation (CTICP_ERR_INVALID_ARGUMENT),
 * unknown dtypes (CTICP_ERR_INVALID_ARGUMENT), more than max_points_per_frame points (CTICP_ERR_CAPACITY). */
int cticp_odometry_register_device(cticp_odometry *h, const cticp_device_scan *scan, void *stream, uint32_t frame_id,
                                   const cticp_frame *initial_estimate,      /* nullable */
                                   const cticp_motion_prior *motion_model,   /* nullable */
                                   cticp_summary *out_summary);
/* cticp_odometry_write_points into a sink in device memory of the handle's device: the same bytes, the same
 * min(capacity_points, count) rule and the same return value. Enqueued on the handle's stream after the work already
 * queued on `stream` (NULL = the legacy default stream), and `stream` is made to wait for it. Returns the count without
 * a host synchronisation. */
int64_t cticp_odometry_write_points_device(cticp_odometry *h, int which, const cticp_cloud_sink *sink, void *stream);

/* ct_icp::Odometry::Trajectory(), src/ct_icp/odometry.cpp:687-689 */
int64_t cticp_odometry_trajectory(cticp_odometry *h, cticp_frame *dst, size_t cap);
/* ct_icp::Odometry::MapSize(), src/ct_icp/odometry.cpp:156-158 */
int64_t cticp_odometry_map_size(cticp_odometry *h);
/* ct_icp::Odometry::GetMapPointCloud(), src/ct_icp/odometry.cpp:692-694 → xyz triples */
int64_t cticp_odometry_map_points(cticp_odometry *h, double *dst_xyz, size_t cap_points);
/* ct_icp::Odometry::Reset(), src/ct_icp/odometry.cpp:956-965 */
int cticp_odometry_reset(cticp_odometry *h);
/* ct_icp::Odometry::Reset(const OdometryOptions&), include/ct_icp/odometry.h:269: same handle, new options (new map) */
int cticp_odometry_reset_options(cticp_odometry *h, const cticp_odometry_options *options);
/* ct_icp::Odometry::GetMapPointer(), src/ct_icp/odometry.cpp:991-993 (borrowed; owned by the odometry) */
cticp_map *cticp_odometry_map(cticp_odometry *h);

/* Snapshots (new): the whole state of a handle — voxel map, trajectory, motion model, robust and insertion counters — as
 * bytes, so that a sequence can be resumed, a map reused and a handle forked. A handle loaded from a snapshot with the
 * saved options registers every later frame exactly as the handle it was saved from (on GPUs with the same SM count).
 * save: dst == NULL returns the size; otherwise writes the snapshot (cap_bytes below the size is refused and nothing is
 * written). Returns the size in bytes or a negative status. Orders itself after all work queued on the handle.
 * Sharded handles: CTICP_ERR_UNSUPPORTED. */
int64_t cticp_odometry_save(cticp_odometry *h, void *dst, size_t cap_bytes);
/* a new handle on `device` from a snapshot; options == NULL: the saved options. Other options may differ from the saved
 * ones only outside map_options and may not need voxel normals the snapshot does not keep (e.g. do_no_insert = 1 to
 * localise against a saved map). A malformed snapshot is CTICP_ERR_INVALID_ARGUMENT, before the device is touched. */
int cticp_odometry_load(const void *src, size_t n_bytes, const cticp_odometry_options *options, int device,
                        cticp_odometry **out);
/* a new handle holding the same state, on `device` (this GPU or another), copied device to device: a direct peer copy
 * when the two GPUs can reach each other, else one the driver stages through host memory */
int cticp_odometry_clone(cticp_odometry *h, int device, cticp_odometry **out);

/* multi-GPU (new; SURVEY §8e): keypoints sharded rank/world, one exchange (sum over ranks) of JTJ/JTr per GN
 * iteration / LM evaluation. unique_id is the 128-byte ncclUniqueId produced by cticp_nccl_unique_id on rank 0 and
 * broadcast by the caller; NCCL bootstraps NVLink peer mailboxes (CUDA IPC) through which the ICP kernels exchange
 * the accumulators themselves, and stays as the fallback (ncclAllReduce per exchange) where peers cannot be mapped. */
int cticp_nccl_unique_id(void *out_128_bytes);
int cticp_odometry_enable_sharding(cticp_odometry *h, const void *unique_id_128_bytes, int rank, int world);
/* 0 = not sharded, 1 = exchange through ncclAllReduce, 2 = in-kernel exchange over peer mailboxes */
int cticp_odometry_sharding_mode(cticp_odometry *h);

/* device timing of the last register_frame (CUDA events on the handle's stream), milliseconds */
typedef struct cticp_device_timing {
    double total_ms;
    double ingest_ms;        /* H2D + sub-sampling + keypoint sampling */
    double icp_ms;           /* all ICP iterations (gather kernel + solve) */
    double gather_ms;        /* neighbor-gather/residual kernel only, summed over iterations */
    double map_update_ms;    /* transform + evict + insert */
    int32_t icp_iterations;
    int32_t kernel_launches;
    uint64_t gather_keypoint_iterations;   /* Σ over iterations of keypoints processed */
    uint64_t gather_stencil_points;        /* Σ S: map points found inside the stencils */
    uint64_t gather_stencil_voxels;        /* Σ (2r+1)^3 probes */
    uint64_t h2d_bytes;                    /* host→device bytes copied by the call (scan + state) */
    uint64_t d2h_bytes;                    /* device→host bytes copied by the call (poses, counters) */
    int32_t gather_launches;               /* launches of the neighbor-gather kernel */
    int32_t icp_batch_groups;              /* problems in the ICP launch of the last frame: 1 solo, B in a grouped launch of
                                              cticp_odometry_register_batch (the frames of its kind: GN, CERES nearest
                                              neighbour, CERES distance-based or ROBUST), 0 without an ICP. With
                                              robust_registration: the launch that ran the frame's last attempt */
} cticp_device_timing;
int cticp_odometry_last_timing(cticp_odometry *h, cticp_device_timing *out);

/* Staged input (new): a scan in host memory can be packed and copied to HBM ahead of time and registered later
 * without any host→device traffic for the points. A scan that is already in device memory (e.g. written by a decoder
 * that runs on the GPU) goes to cticp_odometry_register_device instead.
 * cticp_odometry_stage_frame returns a slot id >= 0; slots live until cticp_odometry_clear_staged. */
int64_t cticp_odometry_stage_frame(cticp_odometry *h, const double *xyz, size_t xyz_stride_bytes, const double *t,
                                   size_t t_stride_bytes, size_t n);
int cticp_odometry_register_staged(cticp_odometry *h, int64_t slot, uint32_t frame_id, cticp_summary *out_summary);

/* ---- one frame on each of many handles in one call ------------------------------------------------------------------
 * Each item registers one frame on its own handle, with the semantics of the single-frame entry its kind names:
 *   CTICP_BATCH_HOST    xyz / t / n with strides in host memory (cticp_odometry_register_frame_ex)
 *   CTICP_BATCH_DEVICE  device_scan + producer stream (cticp_odometry_register_device)
 *   CTICP_BATCH_STAGED  staged_slot (cticp_odometry_register_staged; initial_estimate and motion_model must be NULL)
 * The frames whose single-frame call would run its ICP loop through a persistent kernel with the device tail (k > 0,
 * motion compensation CONTINUOUS, no callback, not sharded, a non-empty scan; solver GN, or solver CERES / ROBUST with
 * options the LM loop accepts) join: the joining frames of each kind — GN, CERES with the nearest-neighbour strategy,
 * CERES with the distance-based strategy, ROBUST — run their loops in ONE grouped launch per kind, each against its own
 * handle's map and options. Frames with robust_registration form four kinds of their own (the same four solvers) and run
 * their attempts in rounds: round r launches attempt r of every such frame still running, one grouped launch per kind;
 * a rejected attempt's next one joins round r + 1. A kind with a single joining frame keeps its solo launch; every
 * other frame takes its single-frame path inside the call. Each item's summary, trajectory entry, map and point vectors
 * are those of the single-frame call, byte for byte when the joining problems of a kind fit on the device together (each
 * gets its solo grid); otherwise they differ by the summation order only and are reproducible from run to run.
 * Errors: CTICP_ERR_INVALID_ARGUMENT before any handle is touched for batch outside [1, 64], a null item, handle, out or
 * scan pointer, an unknown kind, the same handle twice, or handles on different devices; CTICP_ERR_UNSUPPORTED for a
 * sharded handle. Per-item errors (timestamp, capacity, internal, ...) go to that item's status, the other items complete;
 * the call then returns the first failing item's status and cticp_last_error() carries its message.
 * The handles must not be used from other threads during the call. */
enum { CTICP_BATCH_HOST = 0, CTICP_BATCH_DEVICE = 1, CTICP_BATCH_STAGED = 2 };
typedef struct cticp_batch_frame {
    cticp_odometry *handle;
    int32_t kind;                       /* CTICP_BATCH_* */
    uint32_t frame_id;
    /* CTICP_BATCH_HOST */
    const double *xyz;
    size_t xyz_stride_bytes;
    const double *t;
    size_t t_stride_bytes;
    size_t n;
    /* CTICP_BATCH_DEVICE */
    const cticp_device_scan *device_scan;
    void *stream;                       /* the producer's cudaStream_t (NULL: legacy default stream) */
    /* CTICP_BATCH_STAGED */
    int64_t staged_slot;
    const cticp_frame *initial_estimate;        /* nullable */
    const cticp_motion_prior *motion_model;     /* nullable */
    cticp_summary *out;
    int32_t status;                     /* out: CTICP_OK or the item's error */
    int32_t _pad0;
} cticp_batch_frame;
int cticp_odometry_register_batch(cticp_batch_frame *items, size_t batch);
int cticp_odometry_clear_staged(cticp_odometry *h);
/* CUDA-event stopwatch on the handle's stream (the stream every kernel of this handle is launched on) */
int cticp_odometry_timer_start(cticp_odometry *h);
int cticp_odometry_timer_stop(cticp_odometry *h, double *elapsed_ms);   /* synchronises */
/* per-launch CUDA-event timing of the gather kernel (adds two event records per ICP iteration) */
int cticp_odometry_set_gather_timing(cticp_odometry *h, int on);
/* writes `bytes` of device memory (> L2 size flushes the L2) on the handle's stream */
int cticp_odometry_flush_l2(cticp_odometry *h, size_t bytes);

/* ---- Continuous trajectories (slam::LinearContinuousTrajectory, include/SlamCore/trajectory.h:28-130) -----------------
 * A sorted list of poses on one device, the pose at any timestamp, and RawPointsToWorldPoints
 * (src/SlamCore/pointcloud.cxx:313-326) over point records in host or device memory. Build one from
 * cticp_odometry_trajectory: the begin and end pose of every frame. Semantics are the reference's
 * (src/SlamCore/trajectory.cxx), including its quirks:
 *   - Create sorts by (dest_frame_id, dest_timestamp), keeping poses with equal keys in their input order; MaxTimestamp
 *     starts at DBL_MIN (the smallest positive double), as the reference's does.
 *   - lookups clip on bounds: a timestamp with MinTimestamp >= t && t >= MaxTimestamp (sic, trajectory.cxx:58) takes the
 *     first pose when t <= MinTimestamp, else the last; past the last pose, the last pose; a NaN timestamp, pose 0.
 *   - equal lookup indices return that pose unchanged; otherwise alpha is GetAlphaTimestamp (below the pair → 0, above the
 *     pair → 0, equal timestamps → 1) and the pose is slerp (not renormalised) + lerp; dest_timestamp is the lerp of the
 *     two timestamps, dest_frame_id and ref_* come from the lower pose. A point is quat.normalized() * raw + tr of it.
 *   - by frame id: lower_bound on (dest_frame_id, dest_timestamp) and the pose before it; a frame id between the frames
 *     present takes the pair around where it would sort.
 * All arithmetic is fp64, and coordinates and timestamps are read in fp64: no fp32 packing and no alpha rounding (unlike
 * the point vectors of a registration). The device slerp agrees with libm's to the last bit or two. */
typedef struct cticp_trajectory cticp_trajectory;   /* opaque: one device, its own stream */
/* LinearContinuousTrajectory::Create(poses, check_consistency = true). CTICP_ERR_INVALID_ARGUMENT: no poses, a pose whose
 * ref_frame_id differs from the first (sorted) pose's, a timestamp that decreases where dest_frame_id changes, a NaN
 * dest_timestamp. Sorts and uploads the poses and computes the slerp constants of every adjacent pair on the device. */
int cticp_trajectory_create(const cticp_pose *poses, size_t n, int device, cticp_trajectory **out);
void cticp_trajectory_destroy(cticp_trajectory *t);
/* Poses(): the sorted poses; copies min(cap, count), returns the count */
int64_t cticp_trajectory_poses(cticp_trajectory *t, cticp_pose *dst, size_t cap);
/* InterpolatePose(timestamps[i], true) (frame_ids == NULL) or InterpolatePoseWithFrameId(timestamps[i], frame_ids[i],
 * true) of m host timestamps into out[m]. A frame id above every pose's whose query the bounds check does not clip is
 * CTICP_ERR_INVALID_ARGUMENT (the reference's CHECK), and nothing is written. */
int cticp_trajectory_interpolate(cticp_trajectory *t, const double *timestamps, const uint32_t *frame_ids, size_t m,
                                 cticp_pose *out);
/* RawPointsToWorldPoints of the records of `cloud` (host memory; the dtypes, strides and unaligned records that
 * cticp_odometry_register_cloud accepts) into `sink` (host memory, world = 1 required): x, y, z in the world frame as
 * FLOAT32 or FLOAT64 and, when sink->t_dtype != 0, the input timestamp. Writes min(capacity_points, num_points) records
 * and returns num_points. Segments (optional, num_segments = 0 for none): segment s holds points
 * [segment_ends[s-1], segment_ends[s]) of frame segment_frame_ids[s] (segment_ends[-1] = 0) and its points are looked up
 * with that frame id; without segments the lookup is by timestamp. The records and the sink are copied to the device as
 * they are, so the sink's bytes outside its fields are kept; the bytes written are those of cticp_trajectory_transform_device.
 * CTICP_ERR_INVALID_ARGUMENT, before anything is written: null pointers, unknown dtypes, fields outside point_step,
 * sink->world == 0, segment ends that decrease or whose last one is not num_points, a frame id above every pose's. */
int64_t cticp_trajectory_transform(cticp_trajectory *t, const cticp_cloud_view *cloud, const uint64_t *segment_ends,
                                   const uint32_t *segment_frame_ids, size_t num_segments, const cticp_cloud_sink *sink);
/* The same on a scan and a sink in device memory of the trajectory's device: enqueued after the work already queued on
 * `stream` (a cudaStream_t; NULL = the legacy default stream), which is made to wait for the result; no host
 * synchronisation. In addition to the checks above: pointers that are not device memory of the trajectory's device, or
 * a described buffer that extends past its allocation (CTICP_ERR_INVALID_ARGUMENT), checked before anything is enqueued. */
int64_t cticp_trajectory_transform_device(cticp_trajectory *t, const cticp_device_scan *scan, const uint64_t *segment_ends,
                                          const uint32_t *segment_frame_ids, size_t num_segments,
                                          const cticp_cloud_sink *sink, void *stream);

/* ---- Scoring a trajectory against ground truth (include/SlamCore/eval.h, src/SlamCore/eval.cxx) -----------------------
 * kitti::EvaluatePoses and ComputeTrajectoryMetrics on the device, B estimates against one ground truth per call. Each
 * function takes the device first and is synchronous on return. Estimates are num_estimates × n poses, estimate b at
 * est[b * n]. Semantics are the reference's, quirks included:
 *   - KITTI: poses become matrices with quat.normalized(); dist[i] = dist[i-1] + |t[i-1] - t[i]| over the ground truth;
 *     first frames 0, 10, 20, ... < n, and for each one every length in order; the pair ends at the first i >= first with
 *     dist[i] > dist[first] + len (strict: a distance exactly equal does not end it) and is skipped when there is none.
 *     E = (est_f^-1 est_l)^-1 (gt_f^-1 gt_l); t_err = |E.t|, r_err = acos(clamp(0.5 (trace(R_E) - 1), -1, 1)), stored as
 *     (t_err / len, r_err / len), first-frame-major; mean_rpe = 100 sum(t_err / len) / count (NaN for no pair).
 *     ape_i = |(est_i^-1 gt_i).t|; local_i = | |gt_i.t - gt_{i-1}.t| - |est_i.t - est_{i-1}.t| | for i >= 1, its mean
 *     over n - 1 (NaN for n = 1); maxima start at 0 and update on a strict <, index_max_local_err starts at 0.
 *   - metrics: dist[i+1] = dist[i] + |(gt_i.pose.Inverse() * gt_{i+1}.pose).tr| (TSE3 arithmetic); the global
 *     OrthogonalProcrustes (src/SlamCore/geometry.cxx:7-46) of the ground-truth translations onto the estimate's; ate_i =
 *     |quat.normalized() gt_i.t + tr - est_i.t|, max_ate_idx -1 until a value exceeds the running max (from 0, strict >).
 *     Segments form a greedy chain: [start, idx] closes at the first idx with dist[idx] - dist[start] > segment_length,
 *     then start = idx; the trailing part is dropped. A segment of <= 5 poses is skipped (not counted, no fit) but still
 *     advances the chain. Each counted segment gets its own fit and loc_error = the largest |(T_s * gt_i.pose).tr -
 *     est_i.t| over it; segment_mean_ate = sum(loc) / count, segment_mean_ate_ratio = sum(loc / segment_length) / count
 *     (NaN for no counted segment; the reference leaves the ratio's accumulator uninitialised, here it starts at 0).
 *   - a rank-deficient cross-covariance (straight or stationary segments) gives finite metrics; a zero one gives the
 *     identity rotation, as Eigen's JacobiSVD does.
 * The pair selection and the segment chain are exact: both distance arrays are summed in index order with the
 * reference's operation order and no FMA contraction. The other sums are fixed-order block reductions: bit-reproducible
 * from run to run and for each estimate whatever the batch holds, within ~1e-15 relative of a sequential sum.
 * CTICP_ERR_INVALID_ARGUMENT, before anything is written: null pointers (tab_errors / segments may be NULL), n = 0,
 * num_estimates = 0, n <= 5 for the metrics, an empty length list, a length or segment_length that is not finite and
 * > 0, a quaternion that is not finite or is zero, a translation that is not finite, a ground-truth dest_timestamp that
 * is not finite. (Refusing non-finite poses is a deviation: the reference scores them into NaN or undefined behaviour.) */
typedef struct cticp_kitti_errors {   /* kitti::seq_errors without tab_errors and the runner-filled fields */
    double mean_rpe, mean_ape, max_ape, mean_local_err, max_local_err;
    int64_t index_max_local_err;
} cticp_kitti_errors;
typedef struct cticp_traj_segment {   /* slam::segment_t of a counted segment, with its own loc error */
    double segment_length;
    int64_t start_idx, end_idx;       /* inclusive */
    double loc_error;
    double quat[4], tr[3];            /* rigid_transform: estimate ≈ T * ground truth */
} cticp_traj_segment;
typedef struct cticp_traj_metrics {   /* slam::metrics_t without the vectors */
    double total_distance, mean_ate, max_ate;
    int64_t max_ate_idx;
    double segment_mean_ate, segment_mean_ate_ratio;
    int64_t num_segments;
    double quat[4], tr[3];            /* the global rigid_transform */
} cticp_traj_metrics;
/* kitti::EvaluatePoses(gt, est_b, lengths) (eval.cxx:136-178, step size 10) of every estimate. out: num_estimates
 * records. tab_errors (nullable): num_estimates × cap × 2 doubles, estimate b's (t_err / len, r_err / len) pairs at
 * tab_errors[2 * b * cap], min(cap, count) of them. Returns the pair count, which depends on the ground truth only. */
int64_t cticp_kitti_evaluate(int device, const cticp_pose *gt, size_t n, const cticp_pose *est, size_t num_estimates,
                             const double *lengths, size_t num_lengths, cticp_kitti_errors *out, double *tab_errors,
                             size_t cap);
/* kitti::EvaluatePoses(gt, LinearContinuousTrajectory, ...) (eval.cxx:103-111): the estimate is InterpolatePose(
 * gt_i.dest_timestamp, true) of the trajectory, evaluated on the trajectory's device and stream without a host round
 * trip; the same as cticp_kitti_evaluate fed with cticp_trajectory_interpolate's output, bit for bit. */
int64_t cticp_trajectory_kitti_evaluate(cticp_trajectory *t, const cticp_pose *gt, size_t n, const double *lengths,
                                        size_t num_lengths, cticp_kitti_errors *out, double *tab_errors, size_t cap);
/* ComputeTrajectoryMetrics(gt, est_b, segment_length) (eval.cxx:184-291) of every estimate. out: num_estimates records.
 * segments (nullable): num_estimates × cap records, estimate b's counted segments at segments[b * cap], min(cap, count)
 * of them. Returns the number of counted segments, which depends on the ground truth only. */
int64_t cticp_trajectory_metrics(int device, const cticp_pose *gt, size_t n, const cticp_pose *est,
                                 size_t num_estimates, double segment_length, cticp_traj_metrics *out,
                                 cticp_traj_segment *segments, size_t cap);
/* The distances along the ground truth the two functions above select pairs and segments with (metrics_t::distances and
 * the KITTI trajectory_distances): kind 0 = KITTI (matrix translations), kind 1 = ComputeTrajectoryMetrics (TSE3
 * relative poses). out: n doubles. Refusals as above (n >= 1 for both kinds). */
int cticp_trajectory_distances(int device, const cticp_pose *gt, size_t n, int kind, double *out);

/* ---- A dense map of a whole run (slam::SamplePointsInGrid, include/SlamCore/algorithm/grid_sampling.h:12-79) -----------
 * SamplePointsInGrid keeps, per voxel int(p / grid_size) (truncation toward zero, slam::Voxel::Coordinates, so voxel 0
 * spans (-grid_size, grid_size)), the first point that falls into it and then each later one while the voxel holds fewer
 * than num_points_per_voxel points (so 0 and 1 both keep one). The output lists voxel by voxel, in order of first
 * appearance, each voxel's points in input order; max_num_points >= 0 stops it at max_num_points + 1 points (the
 * reference tests size() > max before each push), < 0 means no limit.
 * Two deviations, where the reference has undefined behaviour: a point with a non-finite coordinate or a voxel coordinate
 * outside [-2^20, 2^20) is rejected (not inserted, but counted and numbered), and num_points_per_voxel outside [0, 64]
 * is CTICP_ERR_UNSUPPORTED (a voxel holds at most 64 slots; the reference's negative value means no limit). */
typedef struct cticp_grid_sampling_options {
    double grid_size;               /* 1.0 */
    int32_t num_points_per_voxel;   /* 1 */
    int32_t _pad0;
    int64_t max_num_points;         /* -1 */
} cticp_grid_sampling_options;
void cticp_default_grid_sampling_options(cticp_grid_sampling_options *out);
/* SamplePointsInGrid of n fp64 xyz triples (host memory, stride in bytes) on `device`: the indices kept, min(cap, count)
 * of them into out_indices (nullable); returns the count. CTICP_ERR_INVALID_ARGUMENT for a grid_size that is not finite
 * and > 0 or null pointers; CTICP_ERR_UNSUPPORTED as above. */
int64_t cticp_sample_points_in_grid(int device, const cticp_grid_sampling_options *options, const double *xyz,
                                    size_t stride_bytes, size_t n, uint64_t *out_indices, size_t cap);

/* A world cloud: SamplePointsInGrid grown call by call on one device. After any sequence of adds, an export equals
 * SamplePointsInGrid over the concatenation of every point submitted, in call order, bit for bit: the same points in the
 * same order with the same fp64 values, and each point's source index (its position in that concatenation, rejected
 * points included). Splitting the points into calls, empty ones included, does not change the export; max_num_points
 * applies at export only. Each point is stored in fp64 with its timestamp (0.0 when the input has none).
 * With a trajectory, a point is the world point cticp_trajectory_transform(_device) writes for it (by timestamp, or by
 * frame id with segments), with that function's refusals; without (NULL), the records are world coordinates and may have
 * no timestamp (t_dtype 0). Adds are synchronous on return. Every refusal happens before the cloud changes: null
 * pointers, unknown dtypes, fields outside point_step, device pointers that are not memory of the cloud's device or
 * buffers that end past their allocation, a trajectory or odometry on another device (CTICP_ERR_INVALID_ARGUMENT), more
 * than 2^30 points in one call (CTICP_ERR_INVALID_ARGUMENT), and an add after which the cloud would hold more voxels or
 * points than its capacity (CTICP_ERR_CAPACITY: the cloud stays exactly as it was). */
typedef struct cticp_world_cloud cticp_world_cloud;   /* opaque: one device, its own stream */
typedef struct cticp_world_cloud_stats {
    uint64_t submitted;    /* points of the call */
    uint64_t kept;         /* stored by the call */
    uint64_t rejected;     /* non-finite, or outside the voxel coordinate range */
    uint64_t new_voxels;
} cticp_world_cloud_stats;
/* capacity_voxels 0: clamp(2^22 (0.2 / grid_size)^2, 2^16, 2^26) voxels (16.7M at 0.1 m, 4.2M at 0.2 m);
 * capacity_points 0: capacity_voxels × max(1, num_points_per_voxel). At most 2^30 voxels and 2^32 - 1 points. The
 * device holds ~(44 + 4 max(1, num_points_per_voxel)) bytes per voxel and 40 bytes per point of capacity. */
int cticp_world_cloud_create(const cticp_grid_sampling_options *options, uint64_t capacity_voxels,
                             uint64_t capacity_points, int device, cticp_world_cloud **out);
void cticp_world_cloud_destroy(cticp_world_cloud *wc);
/* host records (the layouts cticp_trajectory_transform reads; t_dtype 0 = no timestamp, without a trajectory only) */
int cticp_world_cloud_add(cticp_world_cloud *wc, cticp_trajectory *trajectory, const cticp_cloud_view *cloud,
                          const uint64_t *segment_ends, const uint32_t *segment_frame_ids, size_t num_segments,
                          cticp_world_cloud_stats *stats_out);
/* device records (scan->t may be NULL with t_dtype 0, without a trajectory only), read after the work queued on `stream`
 * (a cudaStream_t; NULL = the legacy default stream) */
int cticp_world_cloud_add_device(cticp_world_cloud *wc, cticp_trajectory *trajectory, const cticp_device_scan *scan,
                                 const uint64_t *segment_ends, const uint32_t *segment_frame_ids, size_t num_segments,
                                 cticp_world_cloud_stats *stats_out, void *stream);
/* the handle's last CTICP_POINTS_ALL_CORRECTED world points and timestamps, exactly those
 * cticp_odometry_write_points_device writes, device to device */
int cticp_world_cloud_add_odometry(cticp_world_cloud *wc, cticp_odometry *odometry, cticp_world_cloud_stats *stats_out);
int64_t cticp_world_cloud_num_points(cticp_world_cloud *wc);   /* what an export returns (after max_num_points) */
int64_t cticp_world_cloud_num_voxels(cticp_world_cloud *wc);
/* min(capacity_points, num_points) points into a host sink (world = 1 required; sink->data may be NULL to take the
 * source indices only) and, when src_index != NULL, as many source indices; returns num_points */
int64_t cticp_world_cloud_export(cticp_world_cloud *wc, const cticp_cloud_sink *sink, uint64_t *src_index);
/* the same into device memory of the cloud's device, ordered after the work queued on `stream` and before what it queues
 * next, without a host synchronisation */
int64_t cticp_world_cloud_export_device(cticp_world_cloud *wc, const cticp_cloud_sink *sink, uint64_t *src_index,
                                        void *stream);
int cticp_world_cloud_clear(cticp_world_cloud *wc);

/* ---- Neighbourhoods of a point cloud (slam::TNeighborhood, include/SlamCore/experimental/neighborhood.h) -----------------
 * Search: NearestNeighborSearchResult(k, max_radius) + SearchNearestNeighbors. The distance is squared,
 * d2 = ((dx dx + dy dy) + dz dz) with d = query - point, in fp64 without FMA contraction (the bits a host loop gives), and
 * max_radius bounds d2, not the distance: a point is kept only when d2 < max_radius, strictly (nanoflann's leaf test
 * dist < worstDist()). max_radius DBL_MAX (the default) is an unbounded k-nearest search; max_radius <= 0 finds nothing; a
 * NaN max_radius is CTICP_ERR_INVALID_ARGUMENT. The neighbours come ascending by d2, with their count; the reference's bool
 * is count == k. k < 1 is CTICP_ERR_INVALID_ARGUMENT (the reference's CHECK), k > 32 CTICP_ERR_UNSUPPORTED.
 * One deviation: among equal d2, the lower point index comes first (and wins the k-th place); the reference's order there
 * follows its kd-tree traversal.
 * Description: ComputeNeighborhood(values) + ComputeNeighborhoodInfo + ClassifyNeighborhood of a query's k nearest (the
 * query itself included when it is an indexed point) or of a point set. Fewer than 5 points: is_valid 0, every field at its
 * default (scalars -1, vectors 0, type NONE). Otherwise barycenter and covariance are always set, and of the rest only the
 * fields `values` asks for (CTICP_NB_*; the others keep their defaults). line = V.col(0), normal = V.col(2) of the SVD of
 * the covariance, signs unspecified; the singular values are taken as abs before linearity, planarity and a2D; cov_det is
 * Eigen's 3x3 cofactor expansion. A set of coincident points gives NaN (0 / 0) in linearity, planarity and a2D.
 * ClassifyNeighborhood(linearity_threshold, planarity_threshold) (the definition's parameter order; 0.8, 0.8): with both
 * PLANARITY and LINEARITY computed, PLANAR when planarity > its threshold, else LINEAR when linearity > its threshold,
 * else NONE; otherwise VOLUMIC when COV_DET is computed and the neighbourhood has more than 5 points; otherwise NONE.
 * One deviation: the covariance is accumulated centred on the query (on the first point of a point set) instead of the
 * reference's uncentred sum p p^T / n - mu mu^T, which cancels catastrophically at map coordinates of hundreds of metres;
 * the two differ by no more than the reference's own cancellation error.
 * Deviations that replace the reference's aborts: an index of fewer than 5 points is searchable; a point with a
 * non-finite coordinate is rejected when the index is built (it keeps its index, is counted, and is never returned); a
 * query with a non-finite coordinate has 0 neighbours. */
enum {
    CTICP_NB_NO_VALUES = 0,
    CTICP_NB_LINE = 1 << 0,
    CTICP_NB_NORMAL = 1 << 1,
    CTICP_NB_PLANARITY = 1 << 2,
    CTICP_NB_LINEARITY = 1 << 3,
    CTICP_NB_COV_DET = 1 << 4,
    CTICP_NB_KDTREE = 1 << 5,        /* accepted and ignored: every index is searchable */
    CTICP_NB_A2D = 1 << 6,
    CTICP_NB_ALL = 0x7F,
    CTICP_NB_ALL_BUT_KDTREE = 0x5F
};
enum { CTICP_NB_TYPE_NONE = 0, CTICP_NB_TYPE_LINEAR = 1, CTICP_NB_TYPE_PLANAR = 2, CTICP_NB_TYPE_VOLUMIC = 3 };
typedef struct cticp_neighborhood_description {   /* slam::NeighborhoodDescription<double> + is_valid + the class */
    double planarity, linearity, a2D, cov_det;   /* -1 when not computed */
    double line[3], normal[3];                   /* 0 when not computed */
    double barycenter[3];
    double covariance[6];                        /* xx xy xz yy yz zz */
    int32_t is_valid;                            /* at least 5 points */
    int32_t type;                                /* CTICP_NB_TYPE_* */
} cticp_neighborhood_description;
/* The description of num_sets point sets (ComputeNeighborhood(values) then ClassifyNeighborhood) on `device`: set s is the
 * points [segment_ends[s - 1], segment_ends[s]) (from 0) of n fp64 xyz triples in host memory, stride_bytes apart;
 * segment_ends must be non-decreasing and end at n. Refusals (CTICP_ERR_INVALID_ARGUMENT) before anything is written. */
int cticp_neighborhood_describe_sets(int device, const double *xyz, size_t stride_bytes, size_t n,
                                     const uint64_t *segment_ends, size_t num_sets, int values,
                                     double linearity_threshold, double planarity_threshold,
                                     cticp_neighborhood_description *out);
/* An index over one point set on one device (at most 2^31 - 1 points). The points are stored in fp64 in the cells of a
 * uniform grid whose size follows from the data (INTEGRATION.md, "Neighbourhoods and normals of a point cloud"); an
 * index is immutable: rebuild it when its points change. Creation is synchronous. */
typedef struct cticp_neighborhood cticp_neighborhood;   /* opaque: one device, its own stream */
int cticp_neighborhood_create(const double *xyz, size_t stride_bytes, size_t n, int device, cticp_neighborhood **out);
/* a device scan's xyz (float32 or float64; t is ignored), read after the work queued on `stream` */
int cticp_neighborhood_create_device(const cticp_device_scan *scan, void *stream, int device, cticp_neighborhood **out);
/* the points cticp_world_cloud_export returns, in that order (index i = export position i), device to device */
int cticp_neighborhood_create_world_cloud(cticp_world_cloud *wc, cticp_neighborhood **out);
void cticp_neighborhood_destroy(cticp_neighborhood *nb);
int64_t cticp_neighborhood_num_points(cticp_neighborhood *nb);     /* indexed, the rejected ones included */
int64_t cticp_neighborhood_num_rejected(cticp_neighborhood *nb);   /* non-finite points */
/* m queries, fp64 xyz triples (NULL: the indexed points themselves, in index order; m must then be num_points). Writes
 * indices[m k] and d2[m k] (row q: the neighbours of query q ascending by d2, then ~0 and +inf past its count) and
 * counts[m]. Host buffers; synchronous. Refusals before anything is written: null outputs, k, max_radius as above. */
int cticp_neighborhood_search(cticp_neighborhood *nb, const double *queries, size_t m, int k, double max_radius,
                              uint64_t *indices, double *d2, int32_t *counts);
/* the same with the queries and outputs in device memory of the index's device, ordered after the work queued on
 * `stream` and before what it queues next, without a host synchronisation. Buffers that are not memory of that device,
 * end past their allocation, or are not aligned to their scalar (8 bytes; 4 for counts; 8 for descriptions) are
 * CTICP_ERR_INVALID_ARGUMENT. */
int cticp_neighborhood_search_device(cticp_neighborhood *nb, const double *queries, size_t m, int k, double max_radius,
                                     uint64_t *indices, double *d2, int32_t *counts, void *stream);
/* the description of each query's k nearest (within max_radius); with queries = NULL on a world-cloud index, the
 * normals of the whole map, aligned with its export */
int cticp_neighborhood_describe(cticp_neighborhood *nb, const double *queries, size_t m, int k, double max_radius,
                                int values, double linearity_threshold, double planarity_threshold,
                                cticp_neighborhood_description *out);
int cticp_neighborhood_describe_device(cticp_neighborhood *nb, const double *queries, size_t m, int k,
                                       double max_radius, int values, double linearity_threshold,
                                       double planarity_threshold, cticp_neighborhood_description *out, void *stream);

/* ---- Synthetic scenes and sequences (include/SlamCore/experimental/synthetic.h, src/SlamCore/experimental/synthetic.cxx)
 * slam::Scene and slam::SyntheticSensorAcquisition on the device. A scene holds triangles, lines, spheres and balls;
 * primitive index i runs over them in that order, the order every generation emits them in. Semantics are the
 * reference's, quirks included:
 *   - RandomPoint, with draws r uniform on [-1, 1]: triangle weights (r_i + 1)^1.5 over their sum, then sum w_i p_i; line
 *     weights |r_0|, |r_1| over their sum; sphere c + R normalized(r_0..2); ball c + R |r_3| normalized(r_0..2).
 *   - Distance: triangle min(|ptp| + (inside ? 0 : corner/barycentre distance of the plane projection), corner/barycentre
 *     distance of the point), where ptp = (x - p2).Normal(), inside = every coefficient of Eigen's ColPivHouseholderQR
 *     solve of [p0 p1 p2] c = projection lies in [0, 1] (rank-deficient A included: the free coefficients are 0); line:
 *     the projection p0 + sqrt(((x - p0).d)^2) d with d = normalized(p0 - p1), the distance to it plus, outside [p0, p1],
 *     the corner/barycentre distance of the projection, then the min with that of the point; ball max(0, |x - c| - R);
 *     sphere ||x - c| - R|.
 *   - GenerateFrame(n, begin_ts, end_ts, frame_id, d): begin / end = InterpolatePose of the trajectory (clipped on
 *     bounds); a primitive is used when Distance(begin.tr) < d || Distance(end.tr) < d; each of its n points draws its
 *     world point, then alpha = u / RAND_MAX, t = begin.ts (1 - alpha) + alpha end.ts, raw = InterpolatePoseAlpha(begin,
 *     end, alpha).pose.Inverse() * world, and is kept when |raw| < d.
 *   - GeneratePointsCloseToLocation keeps a primitive when Distance(location) <= distance (GeneratePoints: every one).
 * Random numbers: every draw is an integer u in [0, 2^31 - 1] from splitmix64 keyed by (seed, frame id, primitive index,
 * point index, draw index), mapped as Eigen 3.3 maps rand(): -1 + (2 u) / RAND_MAX, and u / RAND_MAX for alpha
 * (RAND_MAX = 2^31 - 1). A frame's points are the same bytes whether it is generated alone or in a batch. The exact
 * key is in DESIGN.md; the reference's process-global rand() stream is not reproduced. */
enum { CTICP_SYN_TRIANGLE = 0, CTICP_SYN_LINE = 1, CTICP_SYN_SPHERE = 2, CTICP_SYN_BALL = 3 };
typedef struct cticp_synthetic_scene cticp_synthetic_scene;   /* opaque: one device, its own stream */
typedef struct cticp_synthetic_frame {   /* one GenerateFrame call */
    double begin_ts, end_ts;
    uint32_t frame_id;
    uint32_t _pad0;
} cticp_synthetic_frame;
/* triangles: 9 doubles each (p0, p1, p2), lines: 6 (p0, p1), spheres and balls: 4 (centre, radius); any array may be NULL
 * when its count is 0. CTICP_ERR_INVALID_ARGUMENT: a non-finite value, a negative radius. The triangles are factored
 * here, once. */
int cticp_synthetic_scene_create(const double *triangles, size_t num_triangles, const double *lines, size_t num_lines,
                                 const double *spheres, size_t num_spheres, const double *balls, size_t num_balls,
                                 int device, cticp_synthetic_scene **out);
void cticp_synthetic_scene_destroy(cticp_synthetic_scene *s);
int64_t cticp_synthetic_scene_num_primitives(cticp_synthetic_scene *s);
/* Distance of m fp64 xyz triples (host) to every primitive: out[q * num_primitives + i]; synchronous */
int cticp_synthetic_scene_distance(cticp_synthetic_scene *s, const double *points, size_t m, double *out);
/* GeneratePoints(n) (location NULL) or GeneratePointsCloseToLocation(n, location, distance): world points as fp64 xyz
 * triples and, when src_index != NULL, (primitive, point) uint32 pairs, min(cap, count) of each. Returns the count. */
int64_t cticp_synthetic_generate_points(cticp_synthetic_scene *s, size_t num_points_per_primitive, const double *location,
                                        double distance, uint64_t seed, double *xyz, size_t cap, uint32_t *src_index);
/* GenerateFrame of m frames, frame k's points after frame k-1's. sink->world selects world (1) or raw (0) coordinates,
 * sink->t_dtype the timestamp; src_index (nullable): (primitive, point) uint32 pairs; frame_ends[m]: frame k's points
 * end at frame_ends[k] (the segment convention of cticp_trajectory_transform). Writes min(capacity_points, count)
 * records and as many pairs; frame_ends hold the full count. Host memory, synchronous; returns the count. The sink's bytes
 * outside its fields are kept. */
int64_t cticp_synthetic_generate_frames(cticp_synthetic_scene *s, cticp_trajectory *t, const cticp_synthetic_frame *frames,
                                        size_t m, size_t num_points_per_primitive, double distance, uint64_t seed,
                                        const cticp_cloud_sink *sink, uint32_t *src_index, uint64_t *frame_ends);
/* The same bytes into device memory of the scene's device (sink, src_index and frame_ends; frames stay on the host),
 * enqueued after the work queued on `stream` (NULL = the legacy default stream), which is made to wait for the result;
 * no host synchronisation, so the count is frame_ends[m - 1] on the device and the call returns CTICP_OK. A frame's slice
 * [frame_ends[k-1], frame_ends[k]) of a world = 0 sink is a cticp_device_scan of that frame for
 * cticp_odometry_register_device.
 * Refusals of both, before anything is written or enqueued: null pointers; a distance that is not finite and > 0;
 * num_points_per_primitive < 2 (the reference's CHECK); a frame with begin_ts > end_ts or a non-finite timestamp; unknown
 * sink dtypes or fields outside point_step; a trajectory on another device (CTICP_ERR_INVALID_ARGUMENT); device pointers
 * that are not memory of the scene's device, end past their allocation or are not aligned (src_index 4, frame_ends 8)
 * (CTICP_ERR_INVALID_ARGUMENT); m × num_primitives × num_points_per_primitive above 2^32 - 1 (CTICP_ERR_CAPACITY). */
int cticp_synthetic_generate_frames_device(cticp_synthetic_scene *s, cticp_trajectory *t,
                                           const cticp_synthetic_frame *frames, size_t m,
                                           size_t num_points_per_primitive, double distance, uint64_t seed,
                                           const cticp_cloud_sink *sink, uint32_t *src_index, uint64_t *frame_ends,
                                           void *stream);
/* SyntheticSensorAcquisition::GeneratePoses(frequency): InterpolatePose of the trajectory at MinTimestamp, then
 * t += 1 / frequency accumulated in fp64 while t <= MaxTimestamp. Writes min(cap, count) poses, returns the count.
 * CTICP_ERR_INVALID_ARGUMENT: a frequency that is not finite and > 0, MaxTimestamp - MinTimestamp <= 1 / frequency (the
 * reference's CHECK). */
int64_t cticp_synthetic_generate_poses(cticp_trajectory *t, double frequency, cticp_pose *out, size_t cap);
/* slam::ApplyUniformNoise of each pose, in place on the host: SE3(AngleAxis_x AngleAxis_y AngleAxis_z, tr) * pose, with
 * angles r_0..2 scale_rot_deg pi / 180 and tr r_3..5 scale_trans_m (the rotation draws first), pose i drawing under key
 * (seed, noise, i). */
int cticp_apply_uniform_noise(cticp_pose *poses, size_t n, double scale_rot_deg, double scale_trans_m, uint64_t seed);

/* ---- Spinning-LiDAR sweeps (a ray-cast scene of a ground plane, axis-aligned boxes and vertical cylinders) --------------
 * A scene holds an optional ground plane z = 0, boxes (x0 y0 z0 x1 y1 z1 mean_free_path; 0 = solid, > 0 = porous) and
 * vertical cylinders (cx cy r h, from z = 0 to h). The range of a ray (origin o, unit direction d, index i in its call,
 * max_range R, 64-bit seed) is the minimum over this candidate set, +INFINITY when it is empty, all in fp64 without FMA:
 *   - ground: -o.z / d.z when d.z < 0 and that is > 0;
 *   - box b (its index in the array as given), unless x1 < o.x - R or x0 > o.x + R: the slab test with the reciprocals
 *     1 / d, fmin / fmax per axis; none when !(tmax >= tmin) or tmin <= 0. A solid box gives tmin; a porous one gives
 *     t = tmin - mfp log(u), u = ((h >> 11) + 0.5) 2^-53, h = splitmix64(seed ^ splitmix64(i 1315423911 + b)) (mod 2^64),
 *     dropped when t > tmax;
 *   - cylinder, unless |cx - o.x| > R: a = dx dx + dy dy, b = 2 (px dx + py dy), c = px px + py py - r r with
 *     p = o - (cx, cy); none when a < 1e-12 or disc = b b - 4 a c <= 0; t = (-b - sqrt(disc)) / (2 a), none when t <= 0 or
 *     z = o.z + t d.z lies outside [0, h].
 * R prunes by x only and does not clip the range: a box inside the x-window may be hit beyond R. The device's log may
 * differ from the host C library's in the last bit, so a porous return may differ by a few ulp; every other range is the
 * host's bit for bit. A ray with a non-finite component gets NaN.
 * Sweeps: rays i = ring n_azimuth + j of a frame (t0, frame_id) point along (cos el cos az, cos el sin az, sin el) in the
 * sensor frame, el = elevations_deg[ring] pi / 180, az = (-2 pi j) / n_azimuth (clockwise), with cos and sin from the host
 * C library; the column's timestamp is t0 + ((j + 0.5) / n_azimuth) period and its pose is the trajectory's
 * InterpolatePose there (cticp_trajectory_interpolate's bits). The ray starts at the pose's translation with the direction
 * quat.normalized() * d_sensor and is cast with seed * 1000003 + frame_id (mod 2^64) and its index i. When
 * noise_sigma > 0 the range gets noise_sigma z, z a Box-Muller normal of two splitmix64 draws keyed by (seed, frame_id, i)
 * (DESIGN.md §5.10 has the key). The ray is kept when the range r is finite and min_range < r < max_range: raw xyz is
 * d_sensor r, world xyz origin + d_world r, the timestamp the column's. Points come in (frame, i) order. */
typedef struct cticp_lidar_scene cticp_lidar_scene;   /* opaque: one device, its own stream */
typedef struct cticp_lidar_sensor {
    const double *elevations_deg;   /* n_rings ring elevations, top to bottom (host memory) */
    uint32_t n_rings, n_azimuth;
    double period;                  /* seconds per revolution */
    double min_range, max_range;    /* the keep bounds (exclusive); max_range is also the cast's R */
    double noise_sigma;             /* >= 0, metres */
} cticp_lidar_sensor;
typedef struct cticp_lidar_frame {   /* one sweep */
    double t0;
    uint32_t frame_id;
    uint32_t _pad0;
} cticp_lidar_frame;
/* boxes: num_boxes × 7 doubles, cylinders: num_cylinders × 4 (either NULL when its count is 0); ground != 0 adds the
 * plane. CTICP_ERR_INVALID_ARGUMENT: a non-finite value, x0 > x1 (or y, z), r < 0, a negative free path. The primitives
 * are binned into a uniform xy grid on the device here, once. */
int cticp_lidar_scene_create(const double *boxes, size_t num_boxes, const double *cylinders, size_t num_cylinders,
                             int ground, int device, cticp_lidar_scene **out);
void cticp_lidar_scene_destroy(cticp_lidar_scene *s);
/* The ranges of n rays (fp64 xyz triples, ray i = index i) into out[n]. Host memory, synchronous. CTICP_ERR_INVALID_ARGUMENT:
 * null pointers, a NaN or non-positive max_range, a non-finite origin or direction component. */
int cticp_lidar_scene_raycast(cticp_lidar_scene *s, const double *origins, const double *directions, size_t n,
                              double max_range, uint64_t seed, double *out);
/* The same on device memory of the scene's device (8-byte aligned, inside their allocations), enqueued after the work
 * queued on `stream` (NULL = the legacy default stream), which is made to wait for the result; no host synchronisation. */
int cticp_lidar_scene_raycast_device(cticp_lidar_scene *s, const double *origins, const double *directions, size_t n,
                                     double max_range, uint64_t seed, double *out, void *stream);
/* m sweeps, frame k's points after frame k-1's. sink->world selects world (1) or raw (0) coordinates, sink->t_dtype the
 * timestamp; ray_index (nullable): each point's ray i; frame_ends[m]: frame k's points end at frame_ends[k]. Writes
 * min(capacity_points, count) records and as many ray indices; frame_ends hold the full count. Host memory, synchronous;
 * returns the count. The sink's bytes outside its fields are kept. A frame is the same bytes alone or in a batch. */
int64_t cticp_lidar_generate_sweeps(cticp_lidar_scene *s, cticp_trajectory *t, const cticp_lidar_sensor *sensor,
                                    const cticp_lidar_frame *frames, size_t m, uint64_t seed,
                                    const cticp_cloud_sink *sink, uint32_t *ray_index, uint64_t *frame_ends);
/* The same bytes into device memory of the scene's device (sink, ray_index and frame_ends; sensor and frames stay on the
 * host), enqueued after the work queued on `stream`, which is made to wait for the result; no host synchronisation, so
 * the count is frame_ends[m - 1] on the device and the call returns CTICP_OK. A frame's slice [frame_ends[k-1],
 * frame_ends[k]) of a world = 0 sink with a timestamp is a cticp_device_scan of that frame for
 * cticp_odometry_register_device.
 * Refusals of both, before anything is written or enqueued: null pointers; n_rings or n_azimuth 0; a non-finite
 * elevation, t0, period or range bound; a NaN or negative noise_sigma; unknown sink dtypes or fields outside point_step;
 * a trajectory on another device (CTICP_ERR_INVALID_ARGUMENT); device pointers that are not memory of the scene's device,
 * end past their allocation or are not aligned (ray_index 4, frame_ends 8) (CTICP_ERR_INVALID_ARGUMENT);
 * m × n_rings × n_azimuth above 2^32 - 1 (CTICP_ERR_CAPACITY). */
int cticp_lidar_generate_sweeps_device(cticp_lidar_scene *s, cticp_trajectory *t, const cticp_lidar_sensor *sensor,
                                       const cticp_lidar_frame *frames, size_t m, uint64_t seed,
                                       const cticp_cloud_sink *sink, uint32_t *ray_index, uint64_t *frame_ends,
                                       void *stream);

/* ---- Dataset sequences (src/ct_icp/dataset.cpp: NCLTIterator, kitti_frame_filter, LoadPoses) ------------------------
 * NCLT velodyne_hits.bin: packets of a 24-byte header (4 x u16 magic 44444, u32 num_hits, u64 utime at byte 12, u32 pad)
 * and num_hits hits of 8 bytes (u16 x, y, z, u8 intensity, u8 laser). A handle copies the bytes into its own device
 * buffer and indexes the packets there: one thread per 8-byte word finds the magic words, the candidates are compacted
 * in order, and each one's successor (c + 24 + 8 num_hits) must be the next candidate; otherwise (a hit whose bytes equal
 * the magic) one device thread walks the packets from offset 0, as the reference reads them. Frame f is packets
 * [f A, (f + 1) A), A = num_aggregated (the reference's nclt_num_aggregated_pc, 220), counted from the start of the bytes.
 * final = 0 keeps whole frames only (bytes_used: where the next chunk starts, so chunking never shifts the grouping);
 * final = 1 lets the last frame hold the complete packets that remain. Decoded points: x = (double) u 0.005 - 100.0 (an
 * fp64 multiply then subtract, no FMA; y, z the same), t = (double) utime in microseconds, in packet then hit order;
 * intensity and laser are dropped. Quirks and deviations:
 *   - a packet with num_hits = 0 counts towards the A packets of its frame but adds no point and no timestamp;
 *   - the sequence ends after the last complete packet (the reference's eof() test reads one header past it);
 *   - a frame's begin time is its first point's timestamp (the reference's minmax of iterators), its end time the
 *     maximum timestamp (the reference dereferences end() there). A frame without points has NaN for both.
 * Refusals at open (CTICP_ERR_INVALID_ARGUMENT, no handle): num_aggregated 0, 32 GiB or more of bytes (the index's
 * counts are 32-bit), a header whose magic is wrong (the message names its byte offset: a refused open returns no handle
 * to read it from), with final = 1 a truncated last packet or trailing bytes. */
typedef struct cticp_nclt cticp_nclt;   /* opaque: one device, its own stream */
typedef struct cticp_nclt_frame {   /* one frame of cticp_nclt_frame_info */
    uint64_t num_points;
    double t_first;                     /* the first point's timestamp (begin_pose) */
    double t_max;                       /* the largest timestamp (end_pose) */
} cticp_nclt_frame;
int cticp_nclt_open(const void *bytes, size_t n_bytes, uint32_t num_aggregated, int final, int device, cticp_nclt **out);
/* the same on bytes in device memory of `device`, read after the work queued on `stream`; returns once indexed */
int cticp_nclt_open_device(const void *bytes, size_t n_bytes, uint32_t num_aggregated, int final, int device,
                           void *stream, cticp_nclt **out);
void cticp_nclt_destroy(cticp_nclt *h);
int64_t cticp_nclt_num_frames(const cticp_nclt *h);
int64_t cticp_nclt_num_packets(const cticp_nclt *h);
int64_t cticp_nclt_num_hits(const cticp_nclt *h);
int64_t cticp_nclt_bytes_used(const cticp_nclt *h);
/* 1 when the index came from the one-thread walk (a chain link failed), 0 when the parallel chain check built it */
int cticp_nclt_index_walked(const cticp_nclt *h);
/* frames [first, first + m) */
int cticp_nclt_frame_info(const cticp_nclt *h, size_t first, size_t m, cticp_nclt_frame *out);
/* The points of frames [first, first + m) into `sink` (world must be 0; t_dtype 0, FLOAT32 or FLOAT64), frame k's ending
 * at frame_ends[k] (counted from the call's first point). Writes min(capacity_points, count) records. Host memory,
 * synchronous; returns the count. CTICP_ERR_INVALID_ARGUMENT before anything is written: frames outside the handle,
 * null pointers, unknown sink dtypes, fields outside point_step, world != 0. */
int64_t cticp_nclt_read_frames(cticp_nclt *h, size_t first, size_t m, const cticp_cloud_sink *sink,
                               uint64_t *frame_ends);
/* The same bytes into device memory of the handle's device (sink and frame_ends, 8-byte aligned), enqueued after the
 * work queued on `stream`, which is made to wait for the result; no host synchronisation. A frame's slice of the sink
 * (with a timestamp) is a cticp_device_scan for cticp_odometry_register_device. */
int cticp_nclt_read_frames_device(cticp_nclt *h, size_t first, size_t m, const cticp_cloud_sink *sink,
                                  uint64_t *frame_ends, void *stream);

/* A binary_little_endian PLY header (PLYSchemaMapper::Builder::BuilderFromPLYFile, src/SlamCore/io.cxx:1234-1325): the
 * "vertex" element's record layout. x, y, z of one float type, each sizeof(scalar) after the previous; the timestamp is
 * the property named "timestamp", "t" or "timestamps" (the first present), of any scalar type (t_dtype 0 when none);
 * point_step is the sum of the property sizes. Host only. CTICP_ERR_UNSUPPORTED: ascii or binary_big_endian, list
 * properties, an element other than vertex. CTICP_ERR_INVALID_ARGUMENT: no "ply" magic or end_header, x, y, z missing,
 * mixed or not consecutive, an unknown property type, a body shorter than num_points records. */
typedef struct cticp_ply_layout {
    uint64_t body_offset;               /* the first record's byte offset */
    uint64_t num_points;
    uint32_t point_step;
    uint32_t xyz_offset;
    int32_t xyz_dtype;                  /* CTICP_DTYPE_FLOAT32 or CTICP_DTYPE_FLOAT64 */
    uint32_t t_offset;
    int32_t t_dtype;                    /* any CTICP_DTYPE_*, 0 = no timestamp */
    int32_t _pad0;
} cticp_ply_layout;
int cticp_ply_layout_parse(const void *bytes, size_t n, cticp_ply_layout *out);

/* kitti_frame_filter (src/ct_icp/dataset.cpp:85-110), one thread per record, in fp64 without FMA: a point with
 * !(z > -5) becomes (0, 0, 0) (NaN points included); any other is rotated by AngleAxis(0.205 pi / 180, axis),
 * axis = (p x (0, 0, 1)).normalized() (a zero axis stays zero, so a point on the z axis is scaled by cos), with Eigen's
 * toRotationMatrix and sin / cos from the host C library. The result is written in the sink's xyz type (the reference
 * writes through its XYZ<double>() proxy into the cloud's own type), with the scan's timestamp when sink->t_dtype != 0.
 * The sink may be the scan's own records (same point_step and xyz offset) with t_dtype = 0: the filter runs in place.
 * Device memory of `device`, enqueued on `stream`. CTICP_ERR_INVALID_ARGUMENT before anything is enqueued: null or
 * out-of-allocation pointers, unknown dtypes, fields outside point_step, world != 0, capacity below the scan's count. */
int cticp_kitti_frame_filter_device(int device, const cticp_device_scan *scan, const cticp_cloud_sink *sink,
                                    void *stream);
/* the same on host records (copied through the device; synchronous) */
int cticp_kitti_frame_filter(int device, const cticp_cloud_view *cloud, const cticp_cloud_sink *sink);

/* Per-frame (min, max) of the scan's timestamps (ProcessFrame's minmax_element, dataset.cpp:306-316): frame k is points
 * [frame_ends[k-1], frame_ends[k]) (frame_ends[-1] = 0) and out_minmax[2k], [2k+1] its range; a frame without points
 * gets (+inf, -inf). A NaN timestamp: the device variant writes (NaN, NaN) for its frame, the host variant returns
 * CTICP_ERR_INVALID_ARGUMENT (the reference's answer depends on the NaN's position). frame_ends must be non-decreasing
 * and end at most at num_points (checked by the host variant; the device one reads them on the device). The scan's
 * x, y, z are not read (scan->xyz may be NULL). */
int cticp_scan_time_ranges_device(int device, const cticp_device_scan *scan, const uint64_t *frame_ends, size_t m,
                                  double *out_minmax, void *stream);
int cticp_scan_time_ranges(int device, const cticp_cloud_view *cloud, const uint64_t *frame_ends, size_t m,
                           double *out_minmax);

/* Ground truth in the LiDAR frame (LoadPoses, dataset.cpp:998-1098). dataset: the reference's DATASET values. Returns
 * the count and copies min(cap, count) poses. Host only.
 *   - KITTI_raw, KITTI, KITTI_360, KITTI_CARLA: LoadPosesKITTIFormat (io.cxx:252-279): each non-empty line's 12 values
 *     fill a 3x4 matrix over the identity, read as `istream >> double` reads them (decimal only: no nan, inf or hex; a
 *     short line keeps the identity's values where it ends; a value that is not a number becomes 0 and ends the line);
 *     Quaternion(R), then CalibI * M * Calib with the sequence's calibration
 *     (KITTI / KITTI_raw: ids 0-2, 3, 4-21; KITTI_360: one; KITTI_CARLA: identity), quaternion normalised;
 *     dest_timestamp (i + 0.5) 0.1 (KITTI_CARLA: i 0.1), dest_frame_id i.
 *   - NCLT: ReadNCLTPoses (:319-381): 7 comma-separated values t, x, y, z, roll, pitch, yaw per line; rotation
 *     Rz(yaw) Ry(pitch) Rx(roll); rows with a NaN skipped; each pose relative to the first, then kNCLT_Calib as above;
 *     dest_frame_id stays 0xFFFFFFFF (the reference's -1). A row of another count or a token that is not a number:
 *     CTICP_ERR_INVALID_ARGUMENT (the reference's CHECK / std::stod).
 *   - HILTI_2021, HILTI_2022 (:642-677): t, x, y, z, qx, qy, qz, qw per line, the quaternion NOT normalised (the
 *     reference discards quat.normalized()), then imu_to_lidar * pose * lidar_to_imu in SE3 arithmetic.
 * One stated deviation: CalibI is the rigid inverse [R^T, -R^T t], where the reference takes Eigen's general
 * Matrix4d::inverse(); the two differ in the last bits, so poses agree with the reference's to ~1e-15, not bit for bit.
 * CTICP_ERR_INVALID_ARGUMENT: a dataset outside these, a KITTI sequence id outside [0, 21]. */
enum { CTICP_DATASET_KITTI_RAW = 0, CTICP_DATASET_KITTI_CARLA = 1, CTICP_DATASET_KITTI = 2, CTICP_DATASET_KITTI_360 = 3,
       CTICP_DATASET_NCLT = 4, CTICP_DATASET_HILTI_2021 = 5, CTICP_DATASET_HILTI_2022 = 6 };
int64_t cticp_ground_truth_parse(int dataset, int sequence_id, const char *text, size_t n, cticp_pose *out, size_t cap);

/* ---- PLY files (slam::WritePLY / WriteCollectionToPLY, src/SlamCore/io.cxx:654-716, over tinyply 2.x) ------------------
 * A file is described as a table of columns: each PLY property is one scalar per item, taken from a strided source and
 * converted to the property's type. The layout is tinyply 2.x's binary writer:
 *     ply\n format binary_little_endian 1.0\n
 *     element <name> <count>\n property <type> <name>\n ...      (per element)
 *     end_header\n
 * then per element `count` packed records, the properties one after the other, no padding. Type names are
 * char uchar short ushort int uint float double. Elements come in order of first appearance in the table (tinyply's
 * add_properties_to_element), properties in table order, and every element of a file has the file's item count (the
 * reference's writer always gives every element kNumItems).
 * Conversions are static_cast as g++ on x86-64 computes them: fp64 -> fp32 rounds to nearest even, integer -> integer is
 * modular, integer -> float rounds to nearest, float -> integer truncates toward zero.
 * Deviation: a float -> integer conversion out of the target's range saturates, and NaN gives 0 (undefined behaviour in
 * the reference).
 * CTICP_DTYPE_INT64 / CTICP_DTYPE_UINT64 are source types of cticp_ply_property only (64-bit indices such as a world
 * cloud's source index); PLY has no 64-bit integers, and every other entry point refuses them. */
enum { CTICP_DTYPE_INT64 = 9, CTICP_DTYPE_UINT64 = 10 };
typedef struct cticp_ply_property {
    const char *element;        /* PLY element name ("vertex", "pose", ...) */
    const char *name;           /* PLY property name */
    int32_t ply_dtype;          /* CTICP_DTYPE_INT8 .. CTICP_DTYPE_FLOAT64 */
    int32_t src_dtype;          /* CTICP_DTYPE_INT8 .. CTICP_DTYPE_UINT64 */
    const void *src;            /* item 0's scalar (any alignment) */
    uint64_t src_stride_bytes;  /* bytes between items; 0 repeats one scalar */
} cticp_ply_property;
/* One file of num_items items from host sources into host bytes, encoded on `device` (synchronous). Returns the file's
 * size and writes it to `out` only when capacity >= size (capacity 0: a size query; out may then be NULL). */
int64_t cticp_ply_write(int device, const cticp_ply_property *props, size_t n_props, uint64_t num_items, void *out,
                        uint64_t capacity);
/* m files from device sources into device memory, back to back, enqueued on `stream` with no host synchronisation.
 * File k holds items [file_ends[k-1], file_ends[k]) of every column (file_ends[-1] = 0); file_offsets[k] is where it
 * starts in `out` and file_offsets[m] the total size. The first min(capacity, total) bytes are written; with capacity
 * 0 only the offsets are (size once, allocate, encode). file_ends are read on the device: each end is clamped to
 * [previous end, num_items], so a decreasing or oversized end gives a short or empty file and never a read past the
 * sources (deviation: the host readers of frame ends refuse such ends). file_ends / file_offsets 8-byte aligned.
 * Refusals of both variants (CTICP_ERR_INVALID_ARGUMENT, before anything is enqueued): null pointers (out may be NULL
 * when capacity is 0, a source when num_items is 0), n_props 0 or above 32, unknown dtypes, an empty element or property
 * name, one longer than 63 bytes or containing whitespace, the same property twice in an element; device pointers that
 * are not memory of `device` or end past their allocation (a column spans (num_items - 1) stride + size bytes). */
int cticp_ply_write_device(int device, const cticp_ply_property *props, size_t n_props, uint64_t num_items,
                           const uint64_t *file_ends, size_t m, void *out, uint64_t capacity, uint64_t *file_offsets,
                           void *stream);
/* slam::ReadPosesFromPLY (io.cxx:359-410): the properties qx qy qz qw x y z ref_t dest_t ref_fid dest_fid of element
 * "pose", found by name in any order (other elements and properties are skipped). Returns the count and copies
 * min(count, cap) poses. Host only. The nine doubles must be FLOAT64 (the reference's CHECK); deviation: the fids must
 * be int or uint (the reference reinterprets whatever is there as pair<int, int>). CTICP_ERR_UNSUPPORTED: ascii or
 * binary_big_endian, list properties. CTICP_ERR_INVALID_ARGUMENT: a malformed header, a missing property, other
 * types, a body shorter than the header says. */
int64_t cticp_ply_read_poses(const void *bytes, size_t n, cticp_pose *out, size_t cap);

/* ---- Map (L2 boundary; used directly by the parity tests) ---------------------------------------------- */

/* MultipleResolutionVoxelMap(const Options&), include/ct_icp/map.h:136-138 */
int cticp_map_create(const cticp_map_options *options, int device, cticp_map **out);
void cticp_map_destroy(cticp_map *m);
/* InsertPointCloud (world points, given order), include/ct_icp/map.h:153-254,261-293. Deviation: voxel coordinates are
 * kept in 21 bits per axis, so a point that is non-finite or whose voxel coordinate lies outside [-2^20, 2^20) on any axis
 * is skipped (not stored, not counted), where the reference's int voxel would keep it; a search whose stencil reaches
 * outside that range finds no neighbours. The same holds for the odometry's map update. */
int cticp_map_insert(cticp_map *m, const double *xyz, size_t stride_bytes, size_t n);
/* InsertPointCloud(pointcloud, frame_poses, ...) where the begin pose of the source frame matters: per-voxel normals
 * are oriented towards `origin` = frame_poses.front().tr (include/ct_icp/map.h:211-235). cticp_map_insert is the same
 * with origin = (0, 0, 0). */
int cticp_map_insert_from(cticp_map *m, const double *xyz, size_t stride_bytes, size_t n, const double origin[3]);
/* RemoveElementsFarFromLocation, include/ct_icp/map.h:305-322 */
int cticp_map_remove_far(cticp_map *m, const double location[3], double distance);
/* NumPoints(), include/ct_icp/map.h:345 (resolution 0) ; num points of any resolution with map_idx */
int64_t cticp_map_num_points(cticp_map *m, int map_idx);
int64_t cticp_map_num_voxels(cticp_map *m, int map_idx);
/* GetMapPoints(map_idx), include/ct_icp/map.h:354-376: xyz + int32 voxel coords per point (either may be NULL) */
int64_t cticp_map_export(cticp_map *m, int map_idx, double *dst_xyz, int32_t *dst_voxel, size_t cap_points);
/* ComputeNeighborhoods(queries, max_num_neighbors), include/ct_icp/map.h:532-540 (default radius, no normal filter).
 * out_points: n × max_num_neighbors × 3 (farthest first, like RadiusSearchInPlace :508-513), out_counts: n */
int cticp_map_compute_neighborhoods(cticp_map *m, const double *queries_xyz, size_t n, int max_num_neighbors,
                                    double *out_points, int32_t *out_counts);
/* ComputeNeighborhoods(queries, radiuses, max_num_neighbors, nearest_neighbors = true, sensor_location),
 * include/ct_icp/map.h:434-447 → RadiusSearchInPlace :449-514: one radius per query (it selects the resolution and the
 * stencil, :416-432); when sensor_location != NULL and the map's select_valid_normals_direction is set, stored points
 * whose oriented normal faces away from the sensor are skipped (:482-490). Output layout as above. */
int cticp_map_radius_search(cticp_map *m, const double *queries_xyz, const double *radiuses, size_t n,
                            int max_num_neighbors, const double *sensor_location, double *out_points,
                            int32_t *out_counts);
/* ClearMap(), include/ct_icp/map.h:296 */
int cticp_map_clear(cticp_map *m);
/* Snapshots of a map (new): a standalone map or the borrowed map of an odometry (the bytes are the map section of the
 * odometry's snapshot); sizing and refusals as cticp_odometry_save / _load. A loaded map is a new standalone map. */
int64_t cticp_map_save(cticp_map *m, void *dst, size_t cap_bytes);
int cticp_map_load(const void *src, size_t n_bytes, int device, cticp_map **out);

/* ---- Registration (L3 boundary) ------------------------------------------------------------------------- */

/* CT_ICP_Registration::Register(map, keypoints, frame, motion_model, strategy), src/ct_icp/ct_icp.cpp:1026-1037.
 * keypoints[i].world is rewritten (as the reference does through the world_point proxy);
 * frame is in/out; previous_frame (nullable) stands for the PreviousFrameMotionModel state and
 * motion_options for its Options (src/ct_icp/motion_model.cpp:12-61, ct_icp.cpp:885-910). */
int cticp_icp_register(cticp_map *m, const cticp_icp_options *options,
                       const cticp_strategy_options *strategy,
                       cticp_wpoint *keypoints, size_t n,
                       cticp_frame *frame,
                       const cticp_frame *previous_frame,
                       const cticp_motion_model_options *motion_options,
                       cticp_icp_summary *out_summary);

/* B independent CT_ICP_Registration::Register problems (solver GN) against one map, in one persistent launch.
 * options and motion_options are shared; keypoints[b] (n[b] records, world rewritten), frames[b] (in/out) and
 * previous_frames[b] are per problem. previous_frames (nullable) is an array of B nullable pointers: problem b has the
 * PreviousFrameMotionModel prior iff previous_frames && previous_frames[b] && motion_options.
 * Each problem follows the semantics of cticp_icp_register: timestamp check, partial update on failure, world rewrite and
 * summary. Contract: when every problem gets the CTAs a solo call would give it (the problems fit the device together)
 * each result is bit-identical to cticp_icp_register's; otherwise the CTAs are shared in proportion to n[b] and a result
 * differs from the solo one by floating-point summation order only, bit-reproducible from run to run.
 * Errors: CTICP_ERR_INVALID_ARGUMENT for null pointers (keypoints[b] may be NULL when n[b] == 0) or batch outside
 * [1, 64]; CTICP_ERR_UNSUPPORTED for a solver other than GN, max_number_neighbors outside [1, 32], or an engine without
 * the persistent GN loop (CTICP_PERSISTENT=0, -DCTICP_GN_GRID_BARRIERS builds); CTICP_ERR_TIMESTAMP when a keypoint of
 * any problem lies outside its frame (nothing is run and no frame is modified); CTICP_ERR_INTERNAL ("Error During
 * Optimization") when some problem's loop timed out — every problem's outputs are written all the same. */
int cticp_icp_register_batch(cticp_map *m, const cticp_icp_options *options, size_t batch,
                             cticp_wpoint *const *keypoints, const size_t *n, cticp_frame *frames,
                             const cticp_frame *const *previous_frames,
                             const cticp_motion_model_options *motion_options,
                             cticp_icp_summary *out_summaries);

/* cticp_icp_register_batch for every solver, with the neighborhood strategy that solver CERES consults (nullable: the
 * default of cticp_icp_register; GN and ROBUST ignore it, as cticp_icp_register does). GN runs the batch above; CERES and
 * ROBUST run the B problems in one launch of the persistent Levenberg-Marquardt kernel, each on its own group of CTAs
 * separated by barriers of that group alone, so problems that stop after different numbers of iterations or evaluations
 * share the launch. Per-problem semantics, the bit-identity contract, the argument checks and the error codes are those
 * of cticp_icp_register_batch; in addition the option checks of cticp_icp_register for CERES / ROBUST run once, before
 * anything is uploaded (CTICP_ERR_UNSUPPORTED: CERES with a distance other than POINT_TO_PLANE, num_closest_neighbors
 * outside [1, min(4, max(min_number_neighbors, 5))], ROBUST with min_number_neighbors < 5, or an engine without the
 * persistent loop (CTICP_PERSISTENT=0); CTICP_ERR_INVALID_ARGUMENT: neighbor count outside [1, 32], a DISTANCE_BASED
 * strategy with radius_max <= 0 or with a normal filter on a map without normals). A problem whose group of CTAs does
 * not meet at a barrier within ~2 s fails alone: CTICP_ERR_INTERNAL after every output is written. */
int cticp_icp_register_batch_ex(cticp_map *m, const cticp_icp_options *options,
                                const cticp_strategy_options *strategy,
                                size_t batch, cticp_wpoint *const *keypoints, const size_t *n, cticp_frame *frames,
                                const cticp_frame *const *previous_frames,
                                const cticp_motion_model_options *motion_options,
                                cticp_icp_summary *out_summaries);

/* Debug tap for parity tests: normal equations of ONE Gauss-Newton linearisation at `frame`
 * (A 12×12 row-major AFTER the 1/n normalisation and regularisers of ct_icp.cpp:877-910, b 12, n used). */
int cticp_icp_gn_normal_equations(cticp_map *m, const cticp_icp_options *options,
                                  const cticp_wpoint *keypoints, size_t n,
                                  const cticp_frame *frame,
                                  const cticp_frame *previous_frame,
                                  const cticp_motion_model_options *motion_options,
                                  double *out_A144, double *out_b12, int32_t *out_num_used);

/* ---- Sampling (a3/a4) ------------------------------------------------------------------------------------ */

/* ct_icp::sub_sample_frame / grid_sampling, src/ct_icp/ct_icp.cpp:65-101, under the order contract
 * (first-seen per voxel of RAW coordinates in the given order; output in order of first appearance).
 * out_indices receives the indices kept; returns the count. */
int64_t cticp_grid_sample_indices(int device, const double *xyz, size_t stride_bytes, size_t n, double voxel_size,
                                  uint32_t *out_indices, size_t cap);
/* The counter-based permutation standing in for std::shuffle: out[perm(i)] = i semantics, see DESIGN.md */
int cticp_permutation(uint64_t seed, uint64_t counter, uint32_t n, uint32_t *out_perm);
/* ct_icp::AdaptiveSamplePointsInGrid, include/ct_icp/algorithm/sampling.h:55-110 (order contract: band by band, first
 * appearance inside a band). out_indices receives the indices kept; returns the count. */
int64_t cticp_adaptive_sample_indices(int device, const cticp_adaptive_options *options, const double *xyz,
                                      size_t stride_bytes, size_t n, uint32_t *out_indices, size_t cap);
void cticp_default_adaptive_options(cticp_adaptive_options *out);

#ifdef __cplusplus
}
#endif
#endif /* CTICP_H */
