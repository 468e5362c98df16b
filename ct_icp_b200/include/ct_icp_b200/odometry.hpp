// ct_icp_b200/odometry.hpp — header-only C++ facade with the API surface of ct_icp::Odometry
// (include/ct_icp/odometry.h:159-402 of the reference) over the C ABI in include/cticp.h.
//
// Same class, method, option and summary field names as the reference, so call sites such as
//   ct_icp::Odometry odometry(options);                                   command/odometry_runner.cpp:154
//   auto summary = odometry.RegisterFrame(frame, frame_id);               command/odometry_runner.cpp:194
//   trajectory.push_back(summary.frame.end_pose);                         command/odometry_runner.cpp:198
//   if (!summary.success) …                                               command/odometry_runner.cpp:276
// compile unchanged — including the slam::PointCloud overloads (any cloud type with size(), XYZConst<double>() and
// TimestampsProxy<double>(), the two views the reference reads, src/ct_icp/odometry.cpp:335-336), the AMotionModel*
// default arguments, RegisterCallback, Reset(options), Map() / MapConst().
// The reference's Eigen / SlamCore types are replaced by minimal PODs with the same member names
// (`pose.quat`, `pose.tr`, `dest_timestamp`, `RawPoint()`, `WorldPoint()`, `Timestamp()`): this header has no
// dependency besides cticp.h. INTEGRATION.md shows the variant that keeps the reference's own headers.
#pragma once
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <map>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "cticp.h"

namespace slam {
typedef unsigned int frame_id_t;

struct Vec3d {   // stand-in for Eigen::Vector3d
    double v[3] = {0, 0, 0};
    double &operator[](int i) { return v[i]; }
    double operator[](int i) const { return v[i]; }
    double &x() { return v[0]; }
    double &y() { return v[1]; }
    double &z() { return v[2]; }
    double x() const { return v[0]; }
    double y() const { return v[1]; }
    double z() const { return v[2]; }
    double norm() const { return std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }
    Vec3d operator-(const Vec3d &o) const { return {{v[0] - o.v[0], v[1] - o.v[1], v[2] - o.v[2]}}; }
};
struct Quatd {   // stand-in for Eigen::Quaterniond (coefficients x, y, z, w)
    double c[4] = {0, 0, 0, 1};
    double x() const { return c[0]; }
    double y() const { return c[1]; }
    double z() const { return c[2]; }
    double w() const { return c[3]; }
    const double *coeffs() const { return c; }
};
struct SE3 {     // slam::TSE3<double>, include/SlamCore/types.h:100-139
    Quatd quat;
    Vec3d tr;
};
struct Pose {    // slam::TPose<double>, include/SlamCore/types.h:162-274
    SE3 pose;
    double ref_timestamp = 0, dest_timestamp = -1;
    frame_id_t ref_frame_id = 0, dest_frame_id = frame_id_t(-1);
    Quatd &QuatRef() { return pose.quat; }
    const Quatd &QuatConstRef() const { return pose.quat; }
    Vec3d &TrRef() { return pose.tr; }
    const Vec3d &TrConstRef() const { return pose.tr; }
};
struct Point3D {
    Vec3d point;
    double timestamp = -1;
};
struct WPoint3D {   // slam::WPoint3D, include/SlamCore/types.h:35-60
    Point3D raw_point;
    Vec3d world_point;
    frame_id_t index_frame = frame_id_t(-1);
    Vec3d &RawPoint() { return raw_point.point; }
    const Vec3d &RawPoint() const { return raw_point.point; }
    Vec3d &WorldPoint() { return world_point; }
    const Vec3d &WorldPoint() const { return world_point; }
    double &Timestamp() { return raw_point.timestamp; }
    const double &Timestamp() const { return raw_point.timestamp; }
};
static_assert(sizeof(WPoint3D) == sizeof(cticp_wpoint), "WPoint3D must keep the reference's 64-byte layout");
}  // namespace slam

namespace ct_icp {

enum CT_ICP_SOLVER { GN = CTICP_SOLVER_GN, CERES = CTICP_SOLVER_CERES, ROBUST = CTICP_SOLVER_ROBUST };
enum LEAST_SQUARES { STANDARD, CAUCHY, HUBER, TOLERANT, TRUNCATED };
enum MOTION_COMPENSATION { NONE = CTICP_MC_NONE, CONSTANT_VELOCITY, ITERATIVE, CONTINUOUS };
enum INITIALIZATION { INIT_NONE, INIT_CONSTANT_VELOCITY };

struct CticpFailure : std::runtime_error {
    int code;
    CticpFailure(int c, const std::string &m) : std::runtime_error(m), code(c) {}
};
inline void cticp_check(int rc) {
    if (rc < 0) throw CticpFailure(rc, cticp_last_error());
}

// ct_icp::CTICPOptions (include/ct_icp/ct_icp.h:56-153): same field names; conversion is a memberwise copy
struct CTICPOptions : cticp_icp_options {
    CTICPOptions() { cticp_default_icp_options(this); }
};

// ct_icp::TrajectoryFrame, include/ct_icp/types.h:31-61
struct TrajectoryFrame {
    slam::Pose begin_pose, end_pose;
    const slam::Vec3d &BeginTr() const { return begin_pose.pose.tr; }
    const slam::Vec3d &EndTr() const { return end_pose.pose.tr; }
    const slam::Quatd &BeginQuat() const { return begin_pose.pose.quat; }
    const slam::Quatd &EndQuat() const { return end_pose.pose.quat; }
};

struct ICPSummary {   // include/ct_icp/ct_icp.h:155-169
    bool success = false;
    int num_residuals_used = 0, num_iters = 0;
    std::string error_log;
    double duration_total = 0, duration_init = 0, avg_duration_iter = 0, avg_duration_neighborhood = 0,
           avg_duration_solve = 0;
};

// ct_icp::OdometryOptions (include/ct_icp/odometry.h:32-157). The polymorphic map_options / neighborhood_strategy
// pointers of the reference are the embedded PODs `map_options` / `neighborhood_strategy`.
struct OdometryOptions : cticp_odometry_options {
    OdometryOptions() { cticp_default_odometry_options(this); }
    static OdometryOptions DefaultDrivingProfile() { OdometryOptions o; cticp_profile_default_driving(&o); return o; }
    static OdometryOptions RobustDrivingProfile() { OdometryOptions o; cticp_profile_robust_driving(&o); return o; }
    static OdometryOptions DefaultRobustOutdoorLowInertia() { OdometryOptions o; cticp_profile_robust_outdoor_low_inertia(&o); return o; }
};

namespace detail {
inline slam::Pose pose_from_c(const cticp_pose &c);
inline cticp_pose pose_to_c(const slam::Pose &p);
}

// ct_icp::AMotionModel / PreviousFrameMotionModel (include/ct_icp/motion_model.h:11-78): the state a caller-owned model
// carries into RegisterFrame. (AddConstraintsToCeresProblem has no meaning off Ceres: the engine adds the same four
// regularisers from `GetOptions()` and the previous frame.)
class AMotionModel {
public:
    virtual ~AMotionModel() = default;
    virtual void UpdateState(const TrajectoryFrame &optimized_frame, int frame_index) = 0;
    virtual void Reset() = 0;
    virtual bool ToPrior(cticp_motion_prior *out) const = 0;   // false: nothing to constrain with yet
};
class PreviousFrameMotionModel : public AMotionModel {
public:
    struct Options : cticp_motion_model_options {
        Options() {
            cticp_odometry_options o;
            cticp_default_odometry_options(&o);
            static_cast<cticp_motion_model_options &>(*this) = o.default_motion_model;
        }
    };
    PreviousFrameMotionModel() = default;
    explicit PreviousFrameMotionModel(const Options &options) : options_(options) {}
    void UpdateState(const TrajectoryFrame &optimized_frame, int) override {
        previous_frame_ = optimized_frame;
        has_frame_ = true;
    }
    void Reset() override { has_frame_ = false; }
    Options &GetOptions() { return options_; }
    const Options &GetOptions() const { return options_; }
    bool ToPrior(cticp_motion_prior *out) const override {
        if (!has_frame_) return false;
        out->options = options_;
        out->previous_frame.begin_pose = detail::pose_to_c(previous_frame_.begin_pose);
        out->previous_frame.end_pose = detail::pose_to_c(previous_frame_.end_pose);
        return true;
    }

private:
    Options options_;
    TrajectoryFrame previous_frame_;
    bool has_frame_ = false;
};

namespace detail {
inline slam::Pose pose_from_c(const cticp_pose &c) {
    slam::Pose p;
    std::memcpy(p.pose.quat.c, c.quat, sizeof(c.quat));
    std::memcpy(p.pose.tr.v, c.tr, sizeof(c.tr));
    p.ref_timestamp = c.ref_timestamp;
    p.dest_timestamp = c.dest_timestamp;
    p.ref_frame_id = c.ref_frame_id;
    p.dest_frame_id = c.dest_frame_id;
    return p;
}
inline cticp_pose pose_to_c(const slam::Pose &p) {
    cticp_pose c;
    std::memcpy(c.quat, p.pose.quat.c, sizeof(c.quat));
    std::memcpy(c.tr, p.pose.tr.v, sizeof(c.tr));
    c.ref_timestamp = p.ref_timestamp;
    c.dest_timestamp = p.dest_timestamp;
    c.ref_frame_id = p.ref_frame_id;
    c.dest_frame_id = p.dest_frame_id;
    return c;
}
inline TrajectoryFrame frame_from_c(const cticp_frame &c) { return {pose_from_c(c.begin_pose), pose_from_c(c.end_pose)}; }
inline cticp_frame frame_to_c(const TrajectoryFrame &f) { return {pose_to_c(f.begin_pose), pose_to_c(f.end_pose)}; }
}  // namespace detail

// ct_icp::ISlamMap view (include/ct_icp/map.h:14-83): the subset callers use through Odometry::GetMapPointer()
class MapView {
public:
    explicit MapView(cticp_map *m) : m_(m) {}
    size_t NumPoints() const { return (size_t) cticp_map_num_points(m_, 0); }                 // map.h:345
    std::vector<slam::Vec3d> MapAsPointCloud() const {                                         // map.h:350
        std::vector<slam::Vec3d> pts(NumPoints());
        if (!pts.empty()) cticp_map_export(m_, 0, &pts[0].v[0], nullptr, pts.size());
        return pts;
    }
    void RemoveElementsFarFromLocation(const slam::Vec3d &location, double distance) {         // map.h:305
        cticp_check(cticp_map_remove_far(m_, location.v, distance));
    }
    cticp_map *handle() const { return m_; }

private:
    cticp_map *m_;
};

class Odometry {
public:
    // The Output of a registration, including metrics (include/ct_icp/odometry.h:163-199)
    struct RegistrationSummary {
        TrajectoryFrame frame, initial_frame;
        int sample_size = 0, number_of_residuals = 0, robust_level = 0;
        double distance_correction = 0.0, relative_distance = 0.0, relative_orientation = 0.0, ego_orientation = 0.0;
        bool success = true, points_added = false;
        int number_of_attempts = 0;
        std::string error_message;
        std::vector<slam::WPoint3D> corrected_points, all_corrected_points, keypoints;
        ICPSummary icp_summary;
        std::map<std::string, double> logged_values;
    };

    // Which of the three point vectors RegisterFrame copies back from the device (the reference always fills all
    // three, odometry.cpp:462-486,597; a caller that only reads the poses can switch the copies off)
    struct CopyBack {
        bool corrected_points = true, all_corrected_points = true, keypoints = true;
    } copy_back;

    // An abstract Callback run at specified stages of the pipeline (include/ct_icp/odometry.h:206-224)
    struct OdometryCallback {
        enum EVENT { BEFORE_ITERATION, ITERATION_COMPLETED, FINISHED_REGISTRATION };
        virtual ~OdometryCallback() = default;
        virtual bool Run(const Odometry &odometry, const std::vector<slam::WPoint3D> &current_frame,
                         const std::vector<slam::WPoint3D> *keypoints = nullptr,
                         const RegistrationSummary *summary = nullptr) = 0;
    };

    explicit Odometry(const OdometryOptions &options, int device = 0) : options_(options) {
        cticp_check(cticp_odometry_create(&options, device, &h_));
        cticp_odometry_set_summary_points(h_, 7);   // the summary carries its three vectors by value: produce them eagerly
    }
    explicit Odometry(const OdometryOptions *options) : Odometry(*options) {}
    ~Odometry() { cticp_odometry_destroy(h_); }
    Odometry(const Odometry &) = delete;
    Odometry &operator=(const Odometry &) = delete;

    // Registers a new Frame to the Map (with custom motion model) (include/ct_icp/odometry.h:231-233). PointCloudT: the
    // reference's slam::PointCloud, or anything with its three accessors (tests/cpp/slam_pointcloud_stub.h)
    template <typename PointCloudT, typename = decltype(std::declval<const PointCloudT &>().template XYZConst<double>())>
    RegistrationSummary RegisterFrame(const PointCloudT &frame, slam::frame_id_t frame_id,
                                      AMotionModel *motion_model = nullptr) {
        return RegisterCloud(frame, frame_id, nullptr, motion_model);
    }
    // … with an initial estimate (:236-239)
    template <typename PointCloudT, typename = decltype(std::declval<const PointCloudT &>().template XYZConst<double>())>
    RegistrationSummary RegisterFrameWithEstimate(const PointCloudT &frame, const TrajectoryFrame &initial_estimate,
                                                  slam::frame_id_t frame_id, AMotionModel *motion_model = nullptr) {
        const cticp_frame est = detail::frame_to_c(initial_estimate);
        return RegisterCloud(frame, frame_id, &est, motion_model);
    }
    // Registers a new Frame to the Map (:242-243)
    RegistrationSummary RegisterFrame(const std::vector<slam::WPoint3D> &frame, AMotionModel *motion_model = nullptr) {
        return Register(frame, nullptr, frame.empty() ? 0 : frame.front().index_frame, motion_model);
    }
    // … with an initial estimate (:246-248)
    RegistrationSummary RegisterFrameWithEstimate(const std::vector<slam::WPoint3D> &frame,
                                                  const TrajectoryFrame &initial_estimate,
                                                  AMotionModel *motion_model = nullptr) {
        const cticp_frame est = detail::frame_to_c(initial_estimate);
        return Register(frame, &est, frame.empty() ? 0 : frame.front().index_frame, motion_model);
    }
    // strided arrays (what the PointCloud overload reads when its fields are already doubles)
    RegistrationSummary RegisterFrame(const double *xyz, size_t xyz_stride_bytes, const double *t,
                                      size_t t_stride_bytes, size_t n, slam::frame_id_t frame_id,
                                      AMotionModel *motion_model = nullptr) {
        return RegisterStrided(xyz, xyz_stride_bytes, t, t_stride_bytes, n, frame_id, nullptr, motion_model);
    }

    // Registers a Callback to the Odometry (:260; src/ct_icp/odometry.cpp:737-750)
    void RegisterCallback(OdometryCallback::EVENT event, OdometryCallback &callback) {
        callbacks_[event].push_back(&callback);
        cticp_check(cticp_odometry_set_callback(h_, &Odometry::Trampoline, this));
    }

    std::vector<TrajectoryFrame> Trajectory() const {   // :251
        const int64_t n = cticp_odometry_trajectory(h_, nullptr, 0);
        std::vector<cticp_frame> raw((size_t) n);
        cticp_odometry_trajectory(h_, raw.data(), raw.size());
        std::vector<TrajectoryFrame> out;
        out.reserve(raw.size());
        for (auto &f : raw) out.push_back(detail::frame_from_c(f));
        return out;
    }
    std::vector<slam::Vec3d> GetMapPointCloud() const { return MapView(cticp_odometry_map(h_)).MapAsPointCloud(); }   // :254
    size_t MapSize() const { return (size_t) cticp_odometry_map_size(h_); }                                           // :258
    MapView &Map() { map_view_ = MapView(cticp_odometry_map(h_)); return map_view_; }                                 // :263 REF_GETTER(Map, *map_)
    const MapView &MapConst() const { map_view_ = MapView(cticp_odometry_map(h_)); return map_view_; }
    void Reset() { cticp_check(cticp_odometry_reset(h_)); }                                                           // :266
    void Reset(const OdometryOptions &options) {                                                                      // :269
        cticp_check(cticp_odometry_reset_options(h_, &options));
        options_ = options;
        cticp_odometry_set_summary_points(h_, SummaryMask());
        if (!callbacks_.empty()) cticp_check(cticp_odometry_set_callback(h_, &Odometry::Trampoline, this));
    }
    std::shared_ptr<MapView> GetMapPointer() { return std::make_shared<MapView>(cticp_odometry_map(h_)); }            // :272
    const OdometryOptions &Options() const { return options_; }
    cticp_odometry *handle() const { return h_; }

    // Snapshots (cticp_odometry_save / _load / _clone): the whole state of the handle as bytes. A handle loaded with the
    // saved options (options == nullptr) registers every later frame exactly as this one would have.
    std::vector<unsigned char> Save() const {
        const int64_t n = cticp_odometry_save(h_, nullptr, 0);
        if (n < 0) cticp_check((int) n);
        std::vector<unsigned char> out((size_t) n);
        const int64_t m = cticp_odometry_save(h_, out.data(), out.size());
        if (m < 0) cticp_check((int) m);
        return out;
    }
    static std::unique_ptr<Odometry> Load(const std::vector<unsigned char> &snapshot, const OdometryOptions *options = nullptr,
                                          int device = 0) {
        cticp_odometry *h = nullptr;
        cticp_check(cticp_odometry_load(snapshot.data(), snapshot.size(), options, device, &h));
        OdometryOptions o;
        if (options) o = *options;
        else std::memcpy(&o, snapshot.data() + kSnapshotHeaderBytes, sizeof(o));   // the options section follows the header
        return std::unique_ptr<Odometry>(new Odometry(h, o));
    }
    std::unique_ptr<Odometry> Clone(int device) const {
        cticp_odometry *h = nullptr;
        cticp_check(cticp_odometry_clone(h_, device, &h));
        return std::unique_ptr<Odometry>(new Odometry(h, options_));
    }

private:
    static constexpr size_t kSnapshotHeaderBytes = 72;   // ct_icp_b200/csrc/snapshot_format.h kHeaderBytes
    Odometry(cticp_odometry *h, const OdometryOptions &options) : h_(h), options_(options) {
        cticp_odometry_set_summary_points(h_, 7);
    }
    int SummaryMask() const {
        return (copy_back.corrected_points ? 1 : 0) | (copy_back.all_corrected_points ? 2 : 0) | (copy_back.keypoints ? 4 : 0);
    }
    RegistrationSummary RegisterStrided(const double *xyz, size_t xyz_stride_bytes, const double *t, size_t t_stride_bytes,
                                        size_t n, slam::frame_id_t frame_id, const cticp_frame *estimate,
                                        AMotionModel *motion_model) {
        if (n == 0) throw std::invalid_argument("The registered frame cannot be empty");
        if (SummaryMask() != last_mask_) {
            cticp_odometry_set_summary_points(h_, SummaryMask());
            last_mask_ = SummaryMask();
        }
        cticp_motion_prior prior;
        const bool with_prior = motion_model && motion_model->ToPrior(&prior);
        cticp_summary s;
        cticp_check(cticp_odometry_register_frame_ex(h_, xyz, xyz_stride_bytes, t, t_stride_bytes, n, frame_id, estimate,
                                                     with_prior ? &prior : nullptr, &s));
        return MakeSummary(s);   // (like the reference, the caller's model is not updated here: the caller calls UpdateState)
    }
    RegistrationSummary Register(const std::vector<slam::WPoint3D> &frame, const cticp_frame *estimate,
                                 slam::frame_id_t frame_id, AMotionModel *motion_model) {
        if (frame.empty()) throw std::invalid_argument("The registered frame cannot be empty");
        return RegisterStrided(frame[0].raw_point.point.v, sizeof(slam::WPoint3D), &frame[0].raw_point.timestamp,
                               sizeof(slam::WPoint3D), frame.size(), frame_id, estimate, motion_model);
    }
    // the reference reads a PointCloud through two converting proxy views (any source scalar type); here they are
    // materialised as doubles once — the zero-copy route for sensor buffers is cticp_odometry_register_cloud
    template <typename PointCloudT>
    RegistrationSummary RegisterCloud(const PointCloudT &frame, slam::frame_id_t frame_id, const cticp_frame *estimate,
                                      AMotionModel *motion_model) {
        const size_t n = frame.size();
        const auto xyz = frame.template XYZConst<double>();
        const auto ts = frame.template TimestampsProxy<double>();
        scratch_.resize(4 * n);
        for (size_t i = 0; i < n; ++i) {
            const auto p = xyz[i];
            scratch_[4 * i] = p[0];
            scratch_[4 * i + 1] = p[1];
            scratch_[4 * i + 2] = p[2];
            scratch_[4 * i + 3] = ts[i];
        }
        return RegisterStrided(scratch_.data(), 32, scratch_.data() + 3, 32, n, frame_id, estimate, motion_model);
    }
    static int Trampoline(int event, void *user) {
        auto *self = static_cast<Odometry *>(user);
        auto it = self->callbacks_.find((typename OdometryCallback::EVENT) event);
        if (it == self->callbacks_.end() || it->second.empty()) return 1;
        std::vector<slam::WPoint3D> frame, keypoints;
        self->FetchAll(CTICP_POINTS_CORRECTED, frame);
        const bool with_kp = event != OdometryCallback::FINISHED_REGISTRATION;   // odometry.cpp:491,568,600
        if (with_kp) self->FetchAll(CTICP_POINTS_KEYPOINTS, keypoints);
        for (auto *cb : it->second)
            if (!cb->Run(*self, frame, with_kp ? &keypoints : nullptr, nullptr)) return 0;   // (:748 passes no summary)
        return 1;
    }
    void FetchAll(int which, std::vector<slam::WPoint3D> &dst) const {
        const int64_t n = cticp_odometry_get_points(h_, which, nullptr, 0);
        dst.resize(n > 0 ? (size_t) n : 0);
        if (n > 0) cticp_odometry_get_points(h_, which, reinterpret_cast<cticp_wpoint *>(dst.data()), dst.size());
    }
    void Fetch(int which, uint64_t count, std::vector<slam::WPoint3D> &dst) {
        dst.resize((size_t) count);
        if (count) cticp_odometry_get_points(h_, which, reinterpret_cast<cticp_wpoint *>(dst.data()), dst.size());
    }
    RegistrationSummary MakeSummary(const cticp_summary &s) {
        RegistrationSummary r;
        r.frame = detail::frame_from_c(s.frame);
        r.initial_frame = detail::frame_from_c(s.initial_frame);
        r.sample_size = s.sample_size;
        r.number_of_residuals = s.number_of_residuals;
        r.robust_level = s.robust_level;
        r.distance_correction = s.distance_correction;
        r.relative_distance = s.relative_distance;
        r.relative_orientation = s.relative_orientation;
        r.ego_orientation = s.ego_orientation;
        r.success = s.success != 0;
        r.points_added = s.points_added != 0;
        r.number_of_attempts = s.number_of_attempts;
        r.error_message = s.error_message;
        r.icp_summary.success = s.icp_summary.success != 0;
        r.icp_summary.num_residuals_used = s.icp_summary.num_residuals_used;
        r.icp_summary.num_iters = s.icp_summary.num_iters;
        r.icp_summary.error_log = s.error_message;
        r.icp_summary.duration_total = s.icp_summary.duration_total;
        r.icp_summary.duration_init = s.icp_summary.duration_init;
        r.icp_summary.avg_duration_iter = s.icp_summary.avg_duration_iter;
        r.icp_summary.avg_duration_neighborhood = s.icp_summary.avg_duration_neighborhood;
        r.icp_summary.avg_duration_solve = s.icp_summary.avg_duration_solve;
        // (all_corrected_points first: the engine sends it back first and in pieces, assembled while the rest is copying)
        if (copy_back.all_corrected_points) Fetch(CTICP_POINTS_ALL_CORRECTED, s.num_all_corrected_points, r.all_corrected_points);
        if (copy_back.keypoints) Fetch(CTICP_POINTS_KEYPOINTS, s.num_keypoints, r.keypoints);
        if (copy_back.corrected_points) Fetch(CTICP_POINTS_CORRECTED, s.num_corrected_points, r.corrected_points);
        // keys the ROS monitor consumes verbatim (ct_icp_odometry_node.cxx:279-287; odometry.cpp:495-513)
        r.logged_values["odometry_total"] = s.odometry_total;                              // :210
        r.logged_values["odometry_initialization"] = s.odometry_initialization;           // :211
        r.logged_values["odometry_total_duration(ms)"] = s.odometry_total;                // :496
        r.logged_values["odometry_initialization(ms)"] = s.odometry_initialization;       // :497
        r.logged_values["odometry_try_register"] = s.odometry_try_register;               // :428
        r.logged_values["odometry_duration_sampling"] = s.odometry_duration_sampling;     // :558
        r.logged_values["odometry_map_update(ms)"] = s.odometry_map_update;               // :498
        r.logged_values["odometry_transform(ms)"] = s.odometry_transform;                 // :499
        r.logged_values["odometry_num_keypoints"] = (double) s.num_keypoints;             // :495
        // LogSummary, :505-513
        r.logged_values["icp_duration_neighborhood"] = s.icp_summary.avg_duration_neighborhood * s.icp_summary.num_iters;
        r.logged_values["icp_duration_solve"] = s.icp_summary.avg_duration_solve * s.icp_summary.num_iters;
        r.logged_values["icp_total_duration"] = s.icp_summary.duration_total;
        r.logged_values["icp_num_iters"] = s.icp_summary.num_iters;
        return r;
    }
    cticp_odometry *h_ = nullptr;
    OdometryOptions options_;
    mutable MapView map_view_{nullptr};
    std::map<typename OdometryCallback::EVENT, std::vector<OdometryCallback *>> callbacks_;
    std::vector<double> scratch_;
    int last_mask_ = 7;
};

}  // namespace ct_icp

namespace slam {

// slam::LinearContinuousTrajectory (include/SlamCore/trajectory.h:28-130) over cticp_trajectory_*: the sorted poses live on
// a device, which evaluates every lookup, interpolation and point transform (semantics: include/cticp.h). Move-only.
class LinearContinuousTrajectory {
public:
    // Create(poses, check_consistency = true) on CUDA device `device`; throws ct_icp::CticpFailure where the reference's
    // CheckConsistency would fail (CTICP_ERR_INVALID_ARGUMENT)
    static LinearContinuousTrajectory Create(std::vector<Pose> &&poses, int device = 0) {
        std::vector<cticp_pose> c;
        c.reserve(poses.size());
        for (const Pose &p : poses) c.push_back(ct_icp::detail::pose_to_c(p));
        LinearContinuousTrajectory t;
        ct_icp::cticp_check(cticp_trajectory_create(c.data(), c.size(), device, &t.h_));
        const int64_t n = cticp_trajectory_poses(t.h_, nullptr, 0);
        c.resize((size_t) n);
        cticp_trajectory_poses(t.h_, c.data(), c.size());
        // Create (trajectory.cxx:170-177): the maximum starts at numeric_limits<double>::min(), as the reference's does
        t.min_ts_ = std::numeric_limits<double>::max();
        t.max_ts_ = std::numeric_limits<double>::min();
        for (const cticp_pose &p : c) {
            t.poses_.push_back(ct_icp::detail::pose_from_c(p));
            if (p.dest_timestamp < t.min_ts_) t.min_ts_ = p.dest_timestamp;
            if (p.dest_timestamp > t.max_ts_) t.max_ts_ = p.dest_timestamp;
        }
        return t;
    }
    LinearContinuousTrajectory(LinearContinuousTrajectory &&o) noexcept
        : h_(std::exchange(o.h_, nullptr)), poses_(std::move(o.poses_)), min_ts_(o.min_ts_), max_ts_(o.max_ts_) {}
    LinearContinuousTrajectory &operator=(LinearContinuousTrajectory &&o) noexcept {
        if (this != &o) {
            if (h_) cticp_trajectory_destroy(h_);
            h_ = std::exchange(o.h_, nullptr);
            poses_ = std::move(o.poses_);
            min_ts_ = o.min_ts_;
            max_ts_ = o.max_ts_;
        }
        return *this;
    }
    LinearContinuousTrajectory(const LinearContinuousTrajectory &) = delete;
    LinearContinuousTrajectory &operator=(const LinearContinuousTrajectory &) = delete;
    ~LinearContinuousTrajectory() {
        if (h_) cticp_trajectory_destroy(h_);
    }

    const std::vector<Pose> &Poses() const { return poses_; }
    double MinTimestamp() const { return min_ts_; }
    double MaxTimestamp() const { return max_ts_; }

    // clip_on_bounds: only true is built (the value every point transform of the reference uses)
    Pose InterpolatePose(double timestamp, bool clip_on_bounds = true) const {
        RequireClip(clip_on_bounds);
        cticp_pose out;
        ct_icp::cticp_check(cticp_trajectory_interpolate(h_, &timestamp, nullptr, 1, &out));
        return ct_icp::detail::pose_from_c(out);
    }
    Pose InterpolatePoseWithFrameId(double timestamp, int frame_id, bool clip_on_bounds = true) const {
        RequireClip(clip_on_bounds);
        const uint32_t fid = (uint32_t) frame_id;
        cticp_pose out;
        ct_icp::cticp_check(cticp_trajectory_interpolate(h_, &timestamp, &fid, 1, &out));
        return ct_icp::detail::pose_from_c(out);
    }
    // TransformPoint (trajectory.cxx:143-155): quat.normalized() * raw + tr of the interpolated pose
    Vec3d TransformPoint(const Vec3d &relative_point, double timestamp) const {
        return Transform(relative_point, timestamp, nullptr);
    }
    Vec3d TransformPoint(const Vec3d &relative_point, double timestamp, int frame_id) const {
        const uint32_t fid = (uint32_t) frame_id;
        return Transform(relative_point, timestamp, &fid);
    }

    cticp_trajectory *Handle() const { return h_; }

private:
    LinearContinuousTrajectory() = default;
    static void RequireClip(bool clip_on_bounds) {
        if (!clip_on_bounds) throw ct_icp::CticpFailure(CTICP_ERR_UNSUPPORTED, "clip_on_bounds = false is not built");
    }
    Vec3d Transform(const Vec3d &p, double t, const uint32_t *fid) const {
        struct {
            double xyz[3], t;
        } rec{{p[0], p[1], p[2]}, t};
        Vec3d w;
        const cticp_cloud_view view{&rec, 1, sizeof(rec), 0, CTICP_DTYPE_FLOAT64, 24, CTICP_DTYPE_FLOAT64, 0};
        const cticp_cloud_sink sink{w.v, 1, sizeof(w.v), 0, CTICP_DTYPE_FLOAT64, 0, 0, 1};
        const uint64_t end = 1;
        const int64_t rc = cticp_trajectory_transform(h_, &view, fid ? &end : nullptr, fid, fid ? 1 : 0, &sink);
        if (rc < 0) ct_icp::cticp_check((int) rc);
        return w;
    }

    cticp_trajectory *h_ = nullptr;
    std::vector<Pose> poses_;
    double min_ts_ = 0, max_ts_ = 0;
};

// PointCloud::RawPointsToWorldPoints(const LinearContinuousTrajectory&) (src/SlamCore/pointcloud.cxx:313-326) on the
// reference's point vector: world_point of every point from its raw point and timestamp, in one device launch. Each run of
// points with the same index_frame is looked up with that frame id (InterpolatePoseWithFrameId), so N scans concatenated
// take each scan's own poses even where two frames share a timestamp.
inline void RawPointsToWorldPoints(std::vector<WPoint3D> &points, const LinearContinuousTrajectory &trajectory) {
    if (points.empty()) return;
    std::vector<uint64_t> ends;
    std::vector<uint32_t> fids;
    for (size_t i = 0; i < points.size(); ++i) {
        if (i > 0 && points[i].index_frame != points[i - 1].index_frame) {
            ends.push_back(i);
            fids.push_back(points[i - 1].index_frame);
        }
    }
    ends.push_back(points.size());
    fids.push_back(points.back().index_frame);
    // the records are read and written in place: raw xyz at 0, timestamp at 24, world xyz at 32 (cticp_wpoint)
    const cticp_cloud_view view{points.data(), points.size(), sizeof(WPoint3D), 0, CTICP_DTYPE_FLOAT64, 24,
                                CTICP_DTYPE_FLOAT64, 0};
    const cticp_cloud_sink sink{points.data(), points.size(), sizeof(WPoint3D), 32, CTICP_DTYPE_FLOAT64, 0, 0, 1};
    const int64_t rc = cticp_trajectory_transform(trajectory.Handle(), &view, ends.data(), fids.data(), ends.size(), &sink);
    if (rc < 0) ct_icp::cticp_check((int) rc);
}

// ---- Scoring against ground truth (include/SlamCore/eval.h) over cticp_kitti_evaluate / cticp_trajectory_metrics -------
// Semantics, quirks and refusals: include/cticp.h. The runner-filled fields keep the reference's defaults.
namespace kitti {

struct errors {
    double t_err;
    double r_err;
    errors() = default;
    errors(double t_err, double r_err) : t_err(t_err), r_err(r_err) {}
};

struct seq_errors {
    std::vector<errors> tab_errors;
    bool success = false;
    bool finished = false;
    double mean_rpe;
    double mean_ape;
    double max_ape;
    double mean_local_err;
    double max_local_err;
    double average_elapsed_ms = -1.0;
    int index_max_local_err;
    double mean_num_attempts;
};

const auto kitti_segment_lengths = std::vector<double>{100., 200., 300., 400., 500., 600., 700., 800.};
const auto indoor_segment_lengths = std::vector<double>{10., 20., 30., 40., 50., 60., 70., 80.};

namespace detail {
inline std::vector<cticp_pose> poses_to_c(const std::vector<Pose> &poses) {
    std::vector<cticp_pose> c;
    c.reserve(poses.size());
    for (const Pose &p : poses) c.push_back(ct_icp::detail::pose_to_c(p));
    return c;
}
// (first frame, length) pairs of ComputeMeanRPE with step size 10: an upper bound of the kept ones
inline size_t max_pairs(size_t n, size_t num_lengths) { return ((n + 9) / 10) * num_lengths; }
inline seq_errors to_seq_errors(const cticp_kitti_errors &e, const std::vector<double> &tab, int64_t count) {
    seq_errors s;
    s.mean_rpe = e.mean_rpe;
    s.mean_ape = e.mean_ape;
    s.max_ape = e.max_ape;
    s.mean_local_err = e.mean_local_err;
    s.max_local_err = e.max_local_err;
    s.index_max_local_err = (int) e.index_max_local_err;
    for (int64_t k = 0; k < count; ++k) s.tab_errors.emplace_back(tab[2 * k], tab[2 * k + 1]);
    return s;
}
}  // namespace detail

// EvaluatePoses(poses_gt, poses_estimated, lengths) (eval.cxx:136-178) on CUDA device `device`
inline seq_errors EvaluatePoses(const std::vector<Pose> &poses_gt, const std::vector<Pose> &poses_estimated,
                                const std::vector<double> &lengths, int device = 0) {
    if (poses_estimated.size() != poses_gt.size())
        throw ct_icp::CticpFailure(CTICP_ERR_INVALID_ARGUMENT, "[ERROR] Couldn't evaluate (all) poses");
    const std::vector<cticp_pose> gt = detail::poses_to_c(poses_gt), est = detail::poses_to_c(poses_estimated);
    const size_t cap = detail::max_pairs(gt.size(), lengths.size());
    std::vector<double> tab(2 * std::max<size_t>(cap, 1));
    cticp_kitti_errors e;
    const int64_t count = cticp_kitti_evaluate(device, gt.data(), gt.size(), est.data(), 1, lengths.data(), lengths.size(),
                                               &e, tab.data(), cap);
    if (count < 0) ct_icp::cticp_check((int) count);
    return detail::to_seq_errors(e, tab, count);
}
inline seq_errors EvaluatePoses(const std::vector<Pose> &poses_gt, const std::vector<Pose> &poses_estimated,
                                bool driving = true, int device = 0) {
    return EvaluatePoses(poses_gt, poses_estimated, driving ? kitti_segment_lengths : indoor_segment_lengths, device);
}
// EvaluatePoses(poses_gt, trajectory) (eval.cxx:103-111): the estimate is trajectory.InterpolatePose(gt_i.dest_timestamp,
// true), interpolated on the trajectory's device
inline seq_errors EvaluatePoses(const std::vector<Pose> &poses_gt, const LinearContinuousTrajectory &trajectory,
                                const std::vector<double> &lengths) {
    const std::vector<cticp_pose> gt = detail::poses_to_c(poses_gt);
    const size_t cap = detail::max_pairs(gt.size(), lengths.size());
    std::vector<double> tab(2 * std::max<size_t>(cap, 1));
    cticp_kitti_errors e;
    const int64_t count = cticp_trajectory_kitti_evaluate(trajectory.Handle(), gt.data(), gt.size(), lengths.data(),
                                                          lengths.size(), &e, tab.data(), cap);
    if (count < 0) ct_icp::cticp_check((int) count);
    return detail::to_seq_errors(e, tab, count);
}
inline seq_errors EvaluatePoses(const std::vector<Pose> &poses_gt, const LinearContinuousTrajectory &trajectory,
                                bool driving = true) {
    return EvaluatePoses(poses_gt, trajectory, driving ? kitti_segment_lengths : indoor_segment_lengths);
}

}  // namespace kitti

struct segment_t {   // slam::segment_t; rigid_transform is set on every counted segment
    double segment_length = 0.;
    size_t start_idx = -1, end_idx = -1;
    std::optional<SE3> rigid_transform;
};

struct metrics_t {   // slam::metrics_t; segment_mean_ate_ratio starts at 0 (the reference leaves it uninitialised)
    std::vector<segment_t> trajectory_segments;
    std::vector<double> loc_errors, distances;
    double segment_mean_ate_ratio = 0., segment_mean_ate = 0.;
    double total_distance = 0.;
    double mean_ate = 0.;
    double max_ate = 0.;
    size_t max_ate_idx = -1;
    std::optional<SE3> rigid_transform;
};

// ComputeTrajectoryMetrics (eval.cxx:184-291) on CUDA device `device`
inline metrics_t ComputeTrajectoryMetrics(const std::vector<Pose> &gt_trajectory, const std::vector<Pose> &trajectory,
                                          double segment_length = 10., int device = 0) {
    if (trajectory.size() != gt_trajectory.size())
        throw ct_icp::CticpFailure(CTICP_ERR_INVALID_ARGUMENT, "the estimate and the ground truth differ in size");
    const std::vector<cticp_pose> gt = kitti::detail::poses_to_c(gt_trajectory), est = kitti::detail::poses_to_c(trajectory);
    const size_t cap = gt.size() > 1 ? std::max<size_t>((gt.size() - 1) / 5, 1) : 1;   // a counted segment spans >= 5 steps
    std::vector<cticp_traj_segment> segs(cap);
    cticp_traj_metrics m;
    const int64_t count = cticp_trajectory_metrics(device, gt.data(), gt.size(), est.data(), 1, segment_length, &m,
                                                   segs.data(), cap);
    if (count < 0) ct_icp::cticp_check((int) count);
    auto se3 = [](const double q[4], const double t[3]) {
        SE3 s;
        for (int k = 0; k < 4; ++k) s.quat.c[k] = q[k];
        for (int k = 0; k < 3; ++k) s.tr[k] = t[k];
        return s;
    };
    metrics_t r;
    r.distances.resize(gt.size());
    ct_icp::cticp_check(cticp_trajectory_distances(device, gt.data(), gt.size(), 1, r.distances.data()));
    r.total_distance = m.total_distance;
    r.mean_ate = m.mean_ate;
    r.max_ate = m.max_ate;
    r.max_ate_idx = (size_t) m.max_ate_idx;
    r.segment_mean_ate = m.segment_mean_ate;
    r.segment_mean_ate_ratio = m.segment_mean_ate_ratio;
    r.rigid_transform = se3(m.quat, m.tr);
    for (int64_t k = 0; k < count; ++k) {
        segment_t s;
        s.segment_length = segs[k].segment_length;
        s.start_idx = (size_t) segs[k].start_idx;
        s.end_idx = (size_t) segs[k].end_idx;
        s.rigid_transform = se3(segs[k].quat, segs[k].tr);
        r.trajectory_segments.push_back(s);
        r.loc_errors.push_back(segs[k].loc_error);
    }
    return r;
}

// ---- A dense map of a whole run (include/SlamCore/algorithm/grid_sampling.h) over cticp_sample_points_in_grid /
// cticp_world_cloud_*. Semantics, quirks, the two deviations and the refusals: include/cticp.h.
struct GridSamplingOptions {
    double grid_size = 1.0;
    int num_points_per_voxel = 1;
    int max_num_points = -1;
};

namespace detail {
inline cticp_grid_sampling_options grid_options_to_c(const GridSamplingOptions &o) {
    cticp_grid_sampling_options c{};
    cticp_default_grid_sampling_options(&c);
    c.grid_size = o.grid_size;
    c.num_points_per_voxel = o.num_points_per_voxel;
    c.max_num_points = o.max_num_points;
    return c;
}
}  // namespace detail

// SamplePointsInGrid(begin, end, options) over points in host memory, on CUDA device `device`: the indices kept, voxel by
// voxel in order of first appearance (the reference walks an unordered_map), each voxel's points in input order
inline std::vector<size_t> SamplePointsInGrid(const std::vector<Vec3d> &points, const GridSamplingOptions &options,
                                              int device = 0) {
    const cticp_grid_sampling_options o = detail::grid_options_to_c(options);
    std::vector<uint64_t> idx(std::max<size_t>(points.size(), 1));
    const int64_t n = cticp_sample_points_in_grid(device, &o, points.empty() ? nullptr : points[0].v, sizeof(Vec3d),
                                                  points.size(), idx.data(), idx.size());
    if (n < 0) ct_icp::cticp_check((int) n);
    return std::vector<size_t>(idx.begin(), idx.begin() + n);
}

// SamplePointsInGrid grown call by call on one device: Points() / SourceIndices() always equal SamplePointsInGrid over
// every point added so far, in call order (world points: the trajectory's RawPointsToWorldPoints of raw ones)
class WorldCloud {
public:
    // capacity 0: the default rule of cticp_world_cloud_create
    explicit WorldCloud(const GridSamplingOptions &options, uint64_t capacity_voxels = 0, uint64_t capacity_points = 0,
                        int device = 0) {
        const cticp_grid_sampling_options o = detail::grid_options_to_c(options);
        ct_icp::cticp_check(cticp_world_cloud_create(&o, capacity_voxels, capacity_points, device, &h_));
    }
    WorldCloud(WorldCloud &&o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
    WorldCloud &operator=(WorldCloud &&o) noexcept {
        if (this != &o) {
            if (h_) cticp_world_cloud_destroy(h_);
            h_ = std::exchange(o.h_, nullptr);
        }
        return *this;
    }
    WorldCloud(const WorldCloud &) = delete;
    WorldCloud &operator=(const WorldCloud &) = delete;
    ~WorldCloud() {
        if (h_) cticp_world_cloud_destroy(h_);
    }

    // world points with their timestamps
    cticp_world_cloud_stats AddWorldPoints(const std::vector<Vec3d> &xyz, const std::vector<double> &timestamps) {
        if (xyz.size() != timestamps.size())
            throw ct_icp::CticpFailure(CTICP_ERR_INVALID_ARGUMENT, "xyz and timestamps must have the same length");
        std::vector<WPoint3D> rec(xyz.size());
        for (size_t i = 0; i < xyz.size(); ++i) {
            rec[i].raw_point.point = xyz[i];
            rec[i].raw_point.timestamp = timestamps[i];
        }
        return AddRecords(rec, nullptr, false);
    }
    // raw points (raw_point, timestamp) placed by the trajectory; each run of equal index_frame is looked up with that
    // frame id, as RawPointsToWorldPoints does
    cticp_world_cloud_stats AddRawPoints(const std::vector<WPoint3D> &points, const LinearContinuousTrajectory &trajectory) {
        return AddRecords(points, trajectory.Handle(), true);
    }
    cticp_world_cloud_stats AddOdometry(cticp_odometry *odometry) {
        cticp_world_cloud_stats st{};
        ct_icp::cticp_check(cticp_world_cloud_add_odometry(h_, odometry, &st));
        return st;
    }
    size_t NumPoints() const { return (size_t) cticp_world_cloud_num_points(h_); }
    size_t NumVoxels() const { return (size_t) cticp_world_cloud_num_voxels(h_); }
    // the cloud as world points with their timestamps (raw_point = world_point) and their source indices
    std::vector<WPoint3D> Points(std::vector<size_t> *source_indices = nullptr) const {
        const size_t n = NumPoints();
        std::vector<WPoint3D> out(n);
        std::vector<uint64_t> src(std::max<size_t>(n, 1));
        const cticp_cloud_sink sink{out.empty() ? nullptr : out.data(), n, sizeof(WPoint3D), 32, CTICP_DTYPE_FLOAT64,
                                    24, CTICP_DTYPE_FLOAT64, 1};
        const int64_t rc = cticp_world_cloud_export(h_, &sink, src.data());
        if (rc < 0) ct_icp::cticp_check((int) rc);
        for (auto &p : out) p.raw_point.point = p.world_point;
        if (source_indices) source_indices->assign(src.begin(), src.begin() + n);
        return out;
    }
    void Clear() { ct_icp::cticp_check(cticp_world_cloud_clear(h_)); }
    cticp_world_cloud *Handle() const { return h_; }

private:
    cticp_world_cloud_stats AddRecords(const std::vector<WPoint3D> &points, cticp_trajectory *traj, bool by_frame) {
        std::vector<uint64_t> ends;
        std::vector<uint32_t> fids;
        if (by_frame && !points.empty()) {
            for (size_t i = 1; i < points.size(); ++i)
                if (points[i].index_frame != points[i - 1].index_frame) {
                    ends.push_back(i);
                    fids.push_back(points[i - 1].index_frame);
                }
            ends.push_back(points.size());
            fids.push_back(points.back().index_frame);
        }
        const cticp_cloud_view view{points.empty() ? nullptr : points.data(), points.size(), sizeof(WPoint3D), 0,
                                    CTICP_DTYPE_FLOAT64, 24, CTICP_DTYPE_FLOAT64, 0};
        cticp_world_cloud_stats st{};
        ct_icp::cticp_check(cticp_world_cloud_add(h_, traj, &view, ends.empty() ? nullptr : ends.data(),
                                                  fids.empty() ? nullptr : fids.data(), ends.size(), &st));
        return st;
    }

    cticp_world_cloud *h_ = nullptr;
};

}  // namespace slam
