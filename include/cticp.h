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

/* ---- Map (L2 boundary; used directly by the parity tests) ---------------------------------------------- */

/* MultipleResolutionVoxelMap(const Options&), include/ct_icp/map.h:136-138 */
int cticp_map_create(const cticp_map_options *options, int device, cticp_map **out);
void cticp_map_destroy(cticp_map *m);
/* InsertPointCloud (world points, given order), include/ct_icp/map.h:153-254,261-293 */
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
