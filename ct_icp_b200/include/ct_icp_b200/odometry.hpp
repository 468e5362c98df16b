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
#include <cstddef>
#include <cstring>
#include <fstream>
#include <iterator>
#include <limits>
#include <map>
#include <memory>
#include <optional>
#include <ostream>
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
    double dot(const Vec3d &o) const { return v[0] * o.v[0] + v[1] * o.v[1] + v[2] * o.v[2]; }
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

// ---- Neighbourhoods of a point cloud (include/SlamCore/experimental/neighborhood.h) over cticp_neighborhood_*.
// Semantics, quirks, the deviations and the refusals: include/cticp.h. Source-compatible with the reference's uses with
// Vec3d in place of Eigen::Vector3d: TNeighborhood(points) (ComputeNeighborhood(ALL)), ComputeNeighborhood(values),
// SearchNearestNeighbors(query, result.ResultSet()), ClassifyNeighborhood(linearity, planarity), description.*.
enum NEIGHBORHOOD_PROPERTIES {
    NO_VALUES = CTICP_NB_NO_VALUES,
    LINE = CTICP_NB_LINE,
    NORMAL = CTICP_NB_NORMAL,
    PLANARITY = CTICP_NB_PLANARITY,
    LINEARITY = CTICP_NB_LINEARITY,
    COV_DET = CTICP_NB_COV_DET,
    KDTREE = CTICP_NB_KDTREE,
    A2D = CTICP_NB_A2D,
    ALL = CTICP_NB_ALL,
    ALL_BUT_KDTREE = CTICP_NB_ALL_BUT_KDTREE
};
enum NEIGHBORHOOD_TYPE { NONE = CTICP_NB_TYPE_NONE, LINEAR, PLANAR, VOLUMIC };

// nanoflann::KNNRadiusResultSet of the reference: k slots and a bound on d2; filled by SearchNearestNeighbors
class KNNRadiusResultSet {
public:
    explicit KNNRadiusResultSet(size_t capacity = 1, double radius = std::numeric_limits<double>::max())
        : max_radius_(radius), capacity_(capacity) {}
    void init(size_t *indices, double *dists) {
        indices_ = indices;
        dists_ = dists;
        count_ = 0;
        if (capacity_) dists_[capacity_ - 1] = std::numeric_limits<double>::max();
    }
    size_t size() const { return count_; }
    bool full() const { return count_ == capacity_; }
    double worstDist() const { return std::min(dists_[capacity_ - 1], max_radius_); }
    size_t capacity() const { return capacity_; }
    double max_radius() const { return max_radius_; }
    // the k nearest as the device found them (ascending by d2, ties by index)
    void assign(const uint64_t *indices, const double *dists, size_t count) {
        for (size_t i = 0; i < count; ++i) {
            indices_[i] = (size_t) indices[i];
            dists_[i] = dists[i];
        }
        count_ = count;
    }

private:
    double max_radius_;
    size_t capacity_, count_ = 0;
    size_t *indices_ = nullptr;
    double *dists_ = nullptr;
};
typedef KNNRadiusResultSet result_set_t;

class NearestNeighborSearchResult {
public:
    // num_neighbors < 1 is the reference's CHECK (CTICP_ERR_INVALID_ARGUMENT); above 32 a search is CTICP_ERR_UNSUPPORTED
    explicit NearestNeighborSearchResult(int num_neighbors = 1,
                                         double max_radius = std::numeric_limits<double>::max()) {
        if (num_neighbors <= 0)
            throw ct_icp::CticpFailure(CTICP_ERR_INVALID_ARGUMENT, "The knn search only works for at least 1 neighbor");
        indices_.resize((size_t) num_neighbors);
        distances_.resize((size_t) num_neighbors);
        result_set_ = KNNRadiusResultSet((size_t) num_neighbors, max_radius);
        result_set_.init(indices_.data(), distances_.data());
    }
    NearestNeighborSearchResult(const NearestNeighborSearchResult &) = delete;   // the result set points into *this
    NearestNeighborSearchResult &operator=(const NearestNeighborSearchResult &) = delete;
    KNNRadiusResultSet &ResultSet() { return result_set_; }
    int NumValidNeighbors() const { return (int) result_set_.size(); }
    std::vector<size_t> Indices() const { return {indices_.begin(), indices_.begin() + NumValidNeighbors()}; }
    std::vector<double> Distances() const { return {distances_.begin(), distances_.begin() + NumValidNeighbors()}; }
    const std::vector<size_t> &AllIndices() const { return indices_; }
    const std::vector<double> &AllDistances() const { return distances_; }

private:
    std::vector<size_t> indices_;
    std::vector<double> distances_;
    KNNRadiusResultSet result_set_;
};

template <typename T>
struct NeighborhoodDescription {
    T planarity = T(-1.0);
    T linearity = T(-1.0);
    T a2D = T(-1);
    T cov_det = T(-1.0);
    Vec3d line, normal, barycenter;
    std::array<std::array<T, 3>, 3> covariance{};
};

struct IdentityConversion {
    const Vec3d &operator()(const Vec3d &p) const { return p; }
};
struct WorldPointConversion {
    const Vec3d &operator()(const WPoint3D &p) const { return p.WorldPoint(); }
};

namespace detail {
inline NeighborhoodDescription<double> description_from_c(const cticp_neighborhood_description &c) {
    NeighborhoodDescription<double> d;
    d.planarity = c.planarity;
    d.linearity = c.linearity;
    d.a2D = c.a2D;
    d.cov_det = c.cov_det;
    for (int a = 0; a < 3; ++a) {
        d.line[a] = c.line[a];
        d.normal[a] = c.normal[a];
        d.barycenter[a] = c.barycenter[a];
    }
    const int ij[6][2] = {{0, 0}, {0, 1}, {0, 2}, {1, 1}, {1, 2}, {2, 2}};
    for (int t = 0; t < 6; ++t) d.covariance[ij[t][0]][ij[t][1]] = d.covariance[ij[t][1]][ij[t][0]] = c.covariance[t];
    return d;
}
}  // namespace detail

// TNeighborhood<SourcePoint, Conversion>: a copy of the points, their description, and a k-nearest index on CUDA
// device `device` (built by ComputeNeighborhood(values & KDTREE), or by the first search: every index is searchable)
template <typename SourcePointT = Vec3d, typename Conversion = IdentityConversion>
struct TNeighborhood {
    typedef std::vector<SourcePointT> vector_points_t;
    static int MinNeighborhoodSize() { return 5; }

    TNeighborhood() = default;
    explicit TNeighborhood(const std::vector<SourcePointT> &pts, int device_ = 0) : points(pts), device(device_) {
        ComputeNeighborhood();
    }

    // the description of the points (fewer than 5: is_valid = false, nothing else changes)
    void ComputeNeighborhood(int values = int(ALL)) {
        if (points.size() < (size_t) MinNeighborhoodSize()) {
            is_valid = false;
            return;
        }
        const std::vector<double> xyz = Packed();
        const uint64_t end = points.size();
        cticp_neighborhood_description c{};
        ct_icp::cticp_check(cticp_neighborhood_describe_sets(device, xyz.data(), 24, points.size(), &end, 1, values,
                                                             0.8, 0.8, &c));
        description = detail::description_from_c(c);
        computed_values = values;
        if (values & KDTREE) BuildIndex();
        is_valid = true;
    }

    // the k nearest of `query` within the result set's bound; true when k were found (nanoflann's result.full())
    bool SearchNearestNeighbors(const Vec3d &query, result_set_t &result_set) {
        const int k = (int) result_set.capacity();
        std::vector<uint64_t> idx((size_t) k);
        std::vector<double> d2((size_t) k);
        int32_t count = 0;
        ct_icp::cticp_check(cticp_neighborhood_search(Index(), query.v, 1, k, result_set.max_radius(), idx.data(),
                                                      d2.data(), &count));
        result_set.assign(idx.data(), d2.data(), (size_t) count);
        return result_set.full();
    }

    // ClassifyNeighborhood(linearity_thresh, planarity_thresh): the definition's parameter order. As in the reference,
    // a neighbourhood with both ratios computed that passes neither leaves `neighborhood` as it was.
    void ClassifyNeighborhood(double linearity_thresh = 0.8, double planarity_thresh = 0.8) {
        if ((computed_values & PLANARITY) && (computed_values & LINEARITY)) {
            if (description.planarity > planarity_thresh) neighborhood = PLANAR;
            else if (description.linearity > linearity_thresh) neighborhood = LINEAR;
        } else if ((computed_values & COV_DET) && points.size() > 5) {
            neighborhood = VOLUMIC;
        } else {
            neighborhood = NONE;
        }
    }

    // batched: the k nearest of every query (row q of indices / d2: k slots, ~0 / +inf past counts[q])
    void SearchNearestNeighbors(const std::vector<Vec3d> &queries, int k, double max_radius,
                                std::vector<uint64_t> &indices, std::vector<double> &d2, std::vector<int32_t> &counts) {
        indices.assign(queries.size() * (size_t) std::max(k, 0), 0);
        d2.assign(indices.size(), 0.0);
        counts.assign(queries.size(), 0);
        ct_icp::cticp_check(cticp_neighborhood_search(Index(), queries.empty() ? nullptr : queries[0].v, queries.size(),
                                                      k, max_radius, indices.data(), d2.data(), counts.data()));
    }
    // batched: ComputeNeighborhood(values) + ClassifyNeighborhood of every query's k nearest (queries empty: every
    // point, in order), with is_valid and the class in each record
    std::vector<cticp_neighborhood_description> DescribeNeighborhoods(
        const std::vector<Vec3d> &queries, int k, double max_radius = std::numeric_limits<double>::max(),
        int values = int(ALL), double linearity_thresh = 0.8, double planarity_thresh = 0.8) {
        const size_t m = queries.empty() ? points.size() : queries.size();
        std::vector<cticp_neighborhood_description> out(m);
        ct_icp::cticp_check(cticp_neighborhood_describe(Index(), queries.empty() ? nullptr : queries[0].v, m, k,
                                                        max_radius, values, linearity_thresh, planarity_thresh,
                                                        out.data()));
        return out;
    }

    NeighborhoodDescription<double> description;
    vector_points_t points;
    int computed_values = NO_VALUES;
    NEIGHBORHOOD_TYPE neighborhood = NONE;
    bool is_valid = false;
    int device = 0;
    std::shared_ptr<cticp_neighborhood> index_;

private:
    std::vector<double> Packed() const {
        Conversion conversion;
        std::vector<double> xyz(3 * std::max<size_t>(points.size(), 1));
        for (size_t i = 0; i < points.size(); ++i)
            for (int a = 0; a < 3; ++a) xyz[3 * i + a] = conversion(points[i])[a];
        return xyz;
    }
    void BuildIndex() {
        const std::vector<double> xyz = Packed();
        cticp_neighborhood *h = nullptr;
        ct_icp::cticp_check(cticp_neighborhood_create(xyz.data(), 24, points.size(), device, &h));
        index_.reset(h, cticp_neighborhood_destroy);
    }
    cticp_neighborhood *Index() {
        if (!index_) BuildIndex();
        return index_.get();
    }
};

typedef TNeighborhood<Vec3d> Neighborhood;
typedef TNeighborhood<WPoint3D, WorldPointConversion> WorldPointNeighborhood;

}  // namespace slam

namespace slam {

// ---- Synthetic scenes and sequences (include/SlamCore/experimental/synthetic.h) over cticp_synthetic_* ----------------
// The reference's primitives, Scene, SyntheticSensorAcquisition and ApplyUniformNoise, with its method names. Every
// Distance and every generation runs on a device (semantics and quirks: include/cticp.h). Where the reference draws from
// the process-global rand(), these draw under the seed member / argument (the draw contract of include/cticp.h), so a
// call is reproducible: the same seed gives the same points. RandomPoint and the YAML readers / writers are not provided.
class Scene;
namespace detail {
// one device scene over the given primitives (created per call: the primitives are plain members the caller may edit)
inline std::shared_ptr<cticp_synthetic_scene> synthetic_scene(const Scene &scene, int device);
}  // namespace detail

class Triangle {
public:
    typedef std::array<Vec3d, 3> PointsArray;
    Triangle() = default;
    Triangle(const PointsArray &array) : points_(array) {}
    PointsArray &Points() { return points_; }
    const PointsArray &Points() const { return points_; }
    Vec3d Normal() const {   // (p0 - p2) x (p1 - p2), normalized
        const Vec3d u = points_[0] - points_[2], v = points_[1] - points_[2];
        Vec3d n{{u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0]}};
        const double z = n[0] * n[0] + n[1] * n[1] + n[2] * n[2];
        if (z > 0)
            for (double &c : n.v) c /= std::sqrt(z);
        return n;
    }
    Vec3d Barycenter() const {
        Vec3d b;
        for (int k = 0; k < 3; ++k) b[k] = (points_[0][k] + points_[1][k] + points_[2][k]) / 3.0;
        return b;
    }
    double Distance(const Vec3d &point, int device = 0) const;
    double ComputeDistance(const Vec3d &point) const { return Distance(point); }

private:
    PointsArray points_;
};

class Line {
public:
    typedef std::array<Vec3d, 2> PointsArray;
    Line() = default;
    Line(const PointsArray &array) : points_(array) {}
    PointsArray &Points() { return points_; }
    const PointsArray &Points() const { return points_; }
    Vec3d Barycenter() const {
        Vec3d b;
        for (int k = 0; k < 3; ++k) b[k] = (points_[0][k] + points_[1][k]) / 2.0;
        return b;
    }
    Vec3d Direction() const {   // (p0 - p1).normalized()
        Vec3d d = points_[0] - points_[1];
        const double z = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
        if (z > 0)
            for (double &c : d.v) c /= std::sqrt(z);
        return d;
    }
    double Distance(const Vec3d &point, int device = 0) const;
    double ComputeDistance(const Vec3d &point) const { return Distance(point); }

private:
    PointsArray points_;
};

// Ball and Sphere: a centre and a radius (1 and the origin by default, as the reference's)
template <int KIND>
class RoundPrimitive {
public:
    RoundPrimitive() = default;
    RoundPrimitive(const Vec3d &center, double radius) : radius_(radius), center_(center) {}
    double &Radius() { return radius_; }
    double Radius() const { return radius_; }
    Vec3d &Center() { return center_; }
    const Vec3d &Center() const { return center_; }
    double Distance(const Vec3d &point, int device = 0) const;
    double ComputeDistance(const Vec3d &point) const { return Distance(point); }

private:
    double radius_ = 1.0;
    Vec3d center_;
};
typedef RoundPrimitive<CTICP_SYN_BALL> Ball;
typedef RoundPrimitive<CTICP_SYN_SPHERE> Sphere;

class Scene {
public:
    size_t NumPrimitives() const { return triangles_.size() + lines_.size() + spheres_.size() + balls_.size(); }
    std::vector<Triangle> &Triangles() { return triangles_; }
    const std::vector<Triangle> &Triangles() const { return triangles_; }
    std::vector<Line> &Lines() { return lines_; }
    const std::vector<Line> &Lines() const { return lines_; }
    std::vector<Sphere> &Spheres() { return spheres_; }
    const std::vector<Sphere> &Spheres() const { return spheres_; }
    std::vector<Ball> &Balls() { return balls_; }
    const std::vector<Ball> &Balls() const { return balls_; }

    std::vector<Vec3d> GeneratePoints(size_t num_points_per_primitive) const {
        return Points(num_points_per_primitive, nullptr, 0.0);
    }
    std::vector<Vec3d> GeneratePointsCloseToLocation(size_t num_points_per_primitive, const Vec3d &location,
                                                     double distance) const {
        return Points(num_points_per_primitive, &location, distance);
    }
    // GenerateSensorPoints between two poses: begin_pose.dest_frame_id keys the draws and is every point's index_frame.
    // The two poses are looked up as a two-pose trajectory, so they must share ref_frame_id and end_pose.dest_timestamp
    // must not lie below begin_pose.dest_timestamp.
    std::vector<WPoint3D> GenerateSensorPoints(size_t num_points_per_primitive, const Pose &begin_pose,
                                               const Pose &end_pose, double distance_to_sensor) const;
    // Distance of every point to every primitive (row q: primitives in generation order), in one launch
    std::vector<double> Distances(const std::vector<Vec3d> &points) const {
        std::vector<double> out(points.size() * NumPrimitives());
        if (out.empty()) return out;
        ct_icp::cticp_check(cticp_synthetic_scene_distance(detail::synthetic_scene(*this, device).get(), points[0].v,
                                                           points.size(), out.data()));
        return out;
    }

    uint64_t seed = 0;   // the draws of every generation of this scene
    int device = 0;

private:
    std::vector<Vec3d> Points(size_t n, const Vec3d *location, double distance) const {
        auto h = detail::synthetic_scene(*this, device);
        const double *loc = location ? location->v : nullptr;
        const int64_t count = cticp_synthetic_generate_points(h.get(), n, loc, distance, seed, nullptr, 0, nullptr);
        if (count < 0) ct_icp::cticp_check((int) count);
        std::vector<Vec3d> out((size_t) count);
        if (count) {
            const int64_t rc = cticp_synthetic_generate_points(h.get(), n, loc, distance, seed, out[0].v, out.size(),
                                                               nullptr);
            if (rc < 0) ct_icp::cticp_check((int) rc);
        }
        return out;
    }

    std::vector<Line> lines_;
    std::vector<Triangle> triangles_;
    std::vector<Ball> balls_;
    std::vector<Sphere> spheres_;
};

namespace detail {
inline std::shared_ptr<cticp_synthetic_scene> synthetic_scene(const Scene &scene, int device) {
    std::vector<double> tri, lin, sph, bal;
    for (const Triangle &t : scene.Triangles())
        for (const Vec3d &p : t.Points()) tri.insert(tri.end(), p.v, p.v + 3);
    for (const Line &l : scene.Lines())
        for (const Vec3d &p : l.Points()) lin.insert(lin.end(), p.v, p.v + 3);
    for (const Sphere &s : scene.Spheres()) {
        sph.insert(sph.end(), s.Center().v, s.Center().v + 3);
        sph.push_back(s.Radius());
    }
    for (const Ball &b : scene.Balls()) {
        bal.insert(bal.end(), b.Center().v, b.Center().v + 3);
        bal.push_back(b.Radius());
    }
    cticp_synthetic_scene *h = nullptr;
    ct_icp::cticp_check(cticp_synthetic_scene_create(tri.data(), scene.Triangles().size(), lin.data(),
                                                     scene.Lines().size(), sph.data(), scene.Spheres().size(),
                                                     bal.data(), scene.Balls().size(), device, &h));
    return std::shared_ptr<cticp_synthetic_scene>(h, cticp_synthetic_scene_destroy);
}
template <typename Fill>
inline double one_primitive_distance(const Vec3d &point, int device, Fill fill) {
    Scene s;
    s.device = device;
    fill(s);
    double d = 0;
    ct_icp::cticp_check(cticp_synthetic_scene_distance(synthetic_scene(s, device).get(), point.v, 1, &d));
    return d;
}
// GenerateFrame of `frames` into the reference's point records: raw xyz and timestamp, then world xyz (the second pass
// keeps the first's bytes), index_frame = the frame's id
inline std::vector<WPoint3D> generate_frames(cticp_synthetic_scene *scene, cticp_trajectory *traj,
                                             const std::vector<cticp_synthetic_frame> &frames, size_t n, double d,
                                             uint64_t seed) {
    std::vector<uint64_t> ends(frames.size());
    cticp_cloud_sink raw{nullptr, 0, sizeof(WPoint3D), 0, CTICP_DTYPE_FLOAT64, 24, CTICP_DTYPE_FLOAT64, 0};
    int64_t count = cticp_synthetic_generate_frames(scene, traj, frames.data(), frames.size(), n, d, seed, &raw, nullptr,
                                                    ends.data());
    if (count < 0) ct_icp::cticp_check((int) count);
    std::vector<WPoint3D> points((size_t) count);
    if (count == 0) return points;
    raw.data = points.data();
    raw.capacity_points = points.size();
    cticp_cloud_sink world{points.data(), points.size(), sizeof(WPoint3D), 32, CTICP_DTYPE_FLOAT64, 0, 0, 1};
    for (const cticp_cloud_sink *sink : {&raw, &world}) {
        count = cticp_synthetic_generate_frames(scene, traj, frames.data(), frames.size(), n, d, seed, sink, nullptr,
                                                ends.data());
        if (count < 0) ct_icp::cticp_check((int) count);
    }
    size_t i = 0;
    for (size_t k = 0; k < frames.size(); ++k)
        for (; i < ends[k]; ++i) points[i].index_frame = frames[k].frame_id;
    return points;
}
}  // namespace detail

inline double Triangle::Distance(const Vec3d &point, int device) const {
    return detail::one_primitive_distance(point, device, [&](Scene &s) { s.Triangles().push_back(*this); });
}
inline double Line::Distance(const Vec3d &point, int device) const {
    return detail::one_primitive_distance(point, device, [&](Scene &s) { s.Lines().push_back(*this); });
}
template <int KIND>
inline double RoundPrimitive<KIND>::Distance(const Vec3d &point, int device) const {
    return detail::one_primitive_distance(point, device, [&](Scene &s) {
        if (KIND == CTICP_SYN_BALL) s.Balls().emplace_back(center_, radius_);
        else s.Spheres().emplace_back(center_, radius_);
    });
}

inline std::vector<WPoint3D> Scene::GenerateSensorPoints(size_t num_points_per_primitive, const Pose &begin_pose,
                                                         const Pose &end_pose, double distance_to_sensor) const {
    std::vector<Pose> two{begin_pose, end_pose};
    two[0].dest_frame_id = 0;   // Create sorts by (dest_frame_id, dest_timestamp): keep begin first
    two[1].dest_frame_id = 1;
    const LinearContinuousTrajectory traj = LinearContinuousTrajectory::Create(std::move(two), device);
    const std::vector<cticp_synthetic_frame> frames{
        {begin_pose.dest_timestamp, end_pose.dest_timestamp, begin_pose.dest_frame_id, 0}};
    return detail::generate_frames(detail::synthetic_scene(*this, device).get(), traj.Handle(), frames,
                                   num_points_per_primitive, distance_to_sensor, seed);
}

class SyntheticSensorAcquisition {
public:
    SyntheticSensorAcquisition(std::shared_ptr<Scene> scene, LinearContinuousTrajectory &&trajectory)
        : scene_(std::move(scene)), base_trajectory_(std::move(trajectory)) {}

    std::shared_ptr<Scene> &GetScene() { return scene_; }
    const std::shared_ptr<Scene> &GetScene() const { return scene_; }
    LinearContinuousTrajectory &GetTrajectory() { return base_trajectory_; }
    const LinearContinuousTrajectory &GetTrajectory() const { return base_trajectory_; }

    // GenerateFrame: begin / end = InterpolatePose(min_timestamp / max_timestamp) of the trajectory
    std::vector<WPoint3D> GenerateFrame(size_t num_points_per_primitive, double min_timestamp, double max_timestamp,
                                        frame_id_t frame_id, double distance_to_sensor) const {
        return GenerateFrames(num_points_per_primitive, {{min_timestamp, max_timestamp, frame_id, 0}}, distance_to_sensor);
    }
    // many GenerateFrame calls in one launch, frame after frame
    std::vector<WPoint3D> GenerateFrames(size_t num_points_per_primitive,
                                         const std::vector<cticp_synthetic_frame> &frames,
                                         double distance_to_sensor) const {
        if (!scene_) throw ct_icp::CticpFailure(CTICP_ERR_INVALID_ARGUMENT, "The scene is not defined");
        return detail::generate_frames(detail::synthetic_scene(*scene_, scene_->device).get(),
                                       base_trajectory_.Handle(), frames, num_points_per_primitive,
                                       distance_to_sensor, scene_->seed);
    }
    std::vector<Pose> GeneratePoses(double frequency = 10) const {
        const int64_t n = cticp_synthetic_generate_poses(base_trajectory_.Handle(), frequency, nullptr, 0);
        if (n < 0) ct_icp::cticp_check((int) n);
        std::vector<cticp_pose> c((size_t) n);
        const int64_t rc = cticp_synthetic_generate_poses(base_trajectory_.Handle(), frequency, c.data(), c.size());
        if (rc < 0) ct_icp::cticp_check((int) rc);
        std::vector<Pose> out;
        for (const cticp_pose &p : c) out.push_back(ct_icp::detail::pose_from_c(p));
        return out;
    }

private:
    std::shared_ptr<Scene> scene_;
    LinearContinuousTrajectory base_trajectory_;
};

// ApplyUniformNoise: SE3(AngleAxis_x AngleAxis_y AngleAxis_z, t) * pose; pose i of the vector draws under key
// (seed, noise, i), a single SE3 under (seed, noise, 0). Host arithmetic; no device needed.
inline void ApplyUniformNoise(std::vector<Pose> &poses, double scale_rot_deg, double scale_trans_m, uint64_t seed = 0) {
    std::vector<cticp_pose> c;
    for (const Pose &p : poses) c.push_back(ct_icp::detail::pose_to_c(p));
    ct_icp::cticp_check(cticp_apply_uniform_noise(c.data(), c.size(), scale_rot_deg, scale_trans_m, seed));
    for (size_t i = 0; i < poses.size(); ++i) poses[i].pose = ct_icp::detail::pose_from_c(c[i]).pose;
}
inline SE3 ApplyUniformNoise(const SE3 &pose, double scale_rot_deg, double scale_trans_m, uint64_t seed = 0) {
    std::vector<Pose> one(1);
    one[0].pose = pose;
    ApplyUniformNoise(one, scale_rot_deg, scale_trans_m, seed);
    return one[0].pose;
}

// ---- Spinning-LiDAR sweeps over cticp_lidar_* -------------------------------------------------------------------------
// A ray-cast scene of a ground plane, axis-aligned boxes (solid or porous) and vertical cylinders, owned on one device,
// with the ranges of given rays and sweeps of a spinning sensor along a trajectory (semantics: include/cticp.h).
struct LidarSensor {
    std::vector<double> elevations_deg;   // one per ring, top to bottom
    uint32_t n_azimuth = 2083;
    double period = 0.1, min_range = 3.0, max_range = 100.0, noise_sigma = 0.0;
};

class LidarScene {
public:
    // boxes: x0 y0 z0 x1 y1 z1 mean_free_path (0 = solid); cylinders: cx cy r h
    LidarScene(const std::vector<std::array<double, 7>> &boxes, const std::vector<std::array<double, 4>> &cylinders,
               bool ground = true, int device = 0) {
        ct_icp::cticp_check(cticp_lidar_scene_create(boxes.empty() ? nullptr : boxes[0].data(), boxes.size(),
                                                     cylinders.empty() ? nullptr : cylinders[0].data(), cylinders.size(),
                                                     ground ? 1 : 0, device, &h_));
    }
    ~LidarScene() {
        if (h_) cticp_lidar_scene_destroy(h_);
    }
    LidarScene(LidarScene &&o) noexcept : h_(o.h_) { o.h_ = nullptr; }
    LidarScene &operator=(LidarScene &&o) noexcept {
        std::swap(h_, o.h_);
        return *this;
    }
    LidarScene(const LidarScene &) = delete;
    LidarScene &operator=(const LidarScene &) = delete;
    cticp_lidar_scene *Handle() const { return h_; }

    // the range of each ray (origin, unit direction; ray i keys the porous draws), +inf where nothing is hit
    std::vector<double> Raycast(const std::vector<Vec3d> &origins, const std::vector<Vec3d> &directions, double max_range,
                                uint64_t seed) const {
        if (origins.size() != directions.size())
            throw ct_icp::CticpFailure(CTICP_ERR_INVALID_ARGUMENT, "origins and directions differ in length");
        std::vector<double> out(origins.size());
        if (!out.empty())
            ct_icp::cticp_check(cticp_lidar_scene_raycast(h_, origins[0].v, directions[0].v, out.size(), max_range, seed,
                                                          out.data()));
        return out;
    }
    // the sweeps of `frames` into the reference's point records: raw xyz and timestamp, world xyz, index_frame = the
    // frame's id; frame_ends (nullable) gets each frame's end
    std::vector<WPoint3D> GenerateSweeps(const LinearContinuousTrajectory &trajectory, const LidarSensor &sensor,
                                         const std::vector<cticp_lidar_frame> &frames, uint64_t seed,
                                         std::vector<uint64_t> *frame_ends = nullptr) const {
        const cticp_lidar_sensor cs{sensor.elevations_deg.data(), (uint32_t) sensor.elevations_deg.size(),
                                    sensor.n_azimuth, sensor.period, sensor.min_range, sensor.max_range,
                                    sensor.noise_sigma};
        std::vector<uint64_t> ends(frames.size());
        cticp_cloud_sink raw{nullptr, 0, sizeof(WPoint3D), 0, CTICP_DTYPE_FLOAT64, 24, CTICP_DTYPE_FLOAT64, 0};
        int64_t count = cticp_lidar_generate_sweeps(h_, trajectory.Handle(), &cs, frames.data(), frames.size(), seed, &raw,
                                                    nullptr, ends.data());
        if (count < 0) ct_icp::cticp_check((int) count);
        std::vector<WPoint3D> points((size_t) count);
        if (count) {
            raw.data = points.data();
            raw.capacity_points = points.size();
            cticp_cloud_sink world{points.data(), points.size(), sizeof(WPoint3D), 32, CTICP_DTYPE_FLOAT64, 0, 0, 1};
            for (const cticp_cloud_sink *sink : {&raw, &world}) {
                count = cticp_lidar_generate_sweeps(h_, trajectory.Handle(), &cs, frames.data(), frames.size(), seed,
                                                    sink, nullptr, ends.data());
                if (count < 0) ct_icp::cticp_check((int) count);
            }
            size_t i = 0;
            for (size_t k = 0; k < frames.size(); ++k)
                for (; i < ends[k]; ++i) points[i].index_frame = frames[k].frame_id;
        }
        if (frame_ends) *frame_ends = ends;
        return points;
    }

private:
    cticp_lidar_scene *h_ = nullptr;
};

}  // namespace slam

// ---- Dataset sequences over cticp_nclt_*, cticp_ply_layout_parse, cticp_kitti_frame_filter, cticp_ground_truth_parse --
// The readers of the reference's dataset.cpp (semantics, quirks and deviations: include/cticp.h, "Dataset sequences").
namespace ct_icp {

// An indexed NCLT velodyne_hits.bin stream on one device: frames of num_aggregated packets
class NCLTHits {
public:
    NCLTHits(const void *bytes, size_t n, uint32_t num_aggregated = 220, bool final = true, int device = 0) {
        cticp_check(cticp_nclt_open(bytes, n, num_aggregated, final ? 1 : 0, device, &h_));
    }
    ~NCLTHits() {
        if (h_) cticp_nclt_destroy(h_);
    }
    NCLTHits(NCLTHits &&o) noexcept : h_(o.h_) { o.h_ = nullptr; }
    NCLTHits &operator=(NCLTHits &&o) noexcept {
        std::swap(h_, o.h_);
        return *this;
    }
    NCLTHits(const NCLTHits &) = delete;
    NCLTHits &operator=(const NCLTHits &) = delete;
    cticp_nclt *Handle() const { return h_; }

    size_t NumFrames() const { return (size_t) Checked(cticp_nclt_num_frames(h_)); }
    size_t NumPackets() const { return (size_t) Checked(cticp_nclt_num_packets(h_)); }
    size_t NumHits() const { return (size_t) Checked(cticp_nclt_num_hits(h_)); }
    size_t BytesUsed() const { return (size_t) Checked(cticp_nclt_bytes_used(h_)); }
    std::vector<cticp_nclt_frame> FrameInfo(size_t first, size_t m) const {
        std::vector<cticp_nclt_frame> out(m);
        cticp_check(cticp_nclt_frame_info(h_, first, m, m ? out.data() : nullptr));
        return out;
    }
    // frames [first, first + m) as the reference's point records: raw xyz and timestamp (microseconds), index_frame = the
    // frame's index in the stream; frame_ends (nullable) gets each frame's end
    std::vector<slam::WPoint3D> ReadFrames(size_t first, size_t m, std::vector<uint64_t> *frame_ends = nullptr) const {
        std::vector<uint64_t> ends(m);
        cticp_cloud_sink sink{nullptr, 0, sizeof(slam::WPoint3D), 0, CTICP_DTYPE_FLOAT64, 24, CTICP_DTYPE_FLOAT64, 0};
        const int64_t count = Checked(cticp_nclt_read_frames(h_, first, m, &sink, m ? ends.data() : nullptr));
        std::vector<slam::WPoint3D> points((size_t) count);
        if (count) {
            sink.data = points.data();
            sink.capacity_points = points.size();
            Checked(cticp_nclt_read_frames(h_, first, m, &sink, ends.data()));
            size_t i = 0;
            for (size_t k = 0; k < m; ++k)
                for (; i < ends[k]; ++i) points[i].index_frame = (slam::frame_id_t) (first + k);
        }
        if (frame_ends) *frame_ends = ends;
        return points;
    }

private:
    static int64_t Checked(int64_t rc) {
        if (rc < 0) cticp_check((int) rc);
        return rc;
    }
    cticp_nclt *h_ = nullptr;
};

// the vertex record layout of a binary_little_endian PLY file (PLYSchemaMapper::Builder::BuilderFromPLYFile's rules)
inline cticp_ply_layout ReadPLYLayout(const void *bytes, size_t n) {
    cticp_ply_layout out{};
    cticp_check(cticp_ply_layout_parse(bytes, n, &out));
    return out;
}

// kitti_frame_filter of the raw points, in place, on `device`
inline void KittiFrameFilter(std::vector<slam::WPoint3D> &points, int device = 0) {
    if (points.empty()) return;
    const cticp_cloud_view view{points.data(), points.size(), sizeof(slam::WPoint3D), 0, CTICP_DTYPE_FLOAT64, 24,
                                CTICP_DTYPE_FLOAT64, 0};
    const cticp_cloud_sink sink{points.data(), points.size(), sizeof(slam::WPoint3D), 0, CTICP_DTYPE_FLOAT64, 0, 0, 0};
    cticp_check(cticp_kitti_frame_filter(device, &view, &sink));
}

// LoadPoses of a ground-truth file's text in the LiDAR frame; dataset is a CTICP_DATASET_* (the reference's DATASET)
inline std::vector<slam::Pose> LoadGroundTruth(int dataset, const std::string &text, int sequence_id = 0) {
    const int64_t n = cticp_ground_truth_parse(dataset, sequence_id, text.data(), text.size(), nullptr, 0);
    if (n < 0) cticp_check((int) n);
    std::vector<cticp_pose> raw((size_t) n);
    if (n) cticp_ground_truth_parse(dataset, sequence_id, text.data(), text.size(), raw.data(), raw.size());
    std::vector<slam::Pose> out(raw.size());
    for (size_t i = 0; i < raw.size(); ++i) {
        for (int k = 0; k < 4; ++k) out[i].pose.quat.c[k] = raw[i].quat[k];
        for (int k = 0; k < 3; ++k) out[i].pose.tr.v[k] = raw[i].tr[k];
        out[i].ref_timestamp = raw[i].ref_timestamp;
        out[i].dest_timestamp = raw[i].dest_timestamp;
        out[i].ref_frame_id = raw[i].ref_frame_id;
        out[i].dest_frame_id = raw[i].dest_frame_id;
    }
    return out;
}

}  // namespace ct_icp

// ---- PLY files over cticp_ply_write, cticp_ply_read_poses -----------------------------------------------------------
// slam::WritePLY / SavePosesAsPLY / ReadPosesFromPLY (src/SlamCore/io.cxx). The file layout, conversions and deviations:
// include/cticp.h, "PLY files". The bytes are encoded on `device`.
namespace slam {

// one PLY property of a WPoint3D file: a scalar at `offset` in each 64-byte record
struct PLYColumn {
    std::string element, name;
    int ply_dtype, src_dtype;
    size_t offset;
};
struct PLYSchemaMapper {
    std::vector<PLYColumn> columns;   // in file order
};

// WPoint3D::FloatSchemaMapper (io.cxx:842-855): vertex x y z timestamp from the raw point, all float
inline PLYSchemaMapper WPoint3DFloatSchema() {
    return {{{"vertex", "x", CTICP_DTYPE_FLOAT32, CTICP_DTYPE_FLOAT64, 0},
             {"vertex", "y", CTICP_DTYPE_FLOAT32, CTICP_DTYPE_FLOAT64, 8},
             {"vertex", "z", CTICP_DTYPE_FLOAT32, CTICP_DTYPE_FLOAT64, 16},
             {"vertex", "timestamp", CTICP_DTYPE_FLOAT32, CTICP_DTYPE_FLOAT64, 24}}};
}
// WPoint3D::DoubleSchemaMapper: the same properties as double
inline PLYSchemaMapper WPoint3DDoubleSchema() {
    PLYSchemaMapper m = WPoint3DFloatSchema();
    for (PLYColumn &c : m.columns) c.ply_dtype = CTICP_DTYPE_FLOAT64;
    return m;
}
// PLYSchemaMapper::BuildDefaultFromSchema(WPoint3D::DefaultSchema()) (types.h:571-590): every property of every
// element, <name> or <name>_<dim>, double except index_frame (uint); elements in the std::map order of
// WriteCollectionToPLY, properties in insertion order
inline PLYSchemaMapper WPoint3DDefaultSchema() {
    struct Property {
        const char *name;
        int type;
        size_t offset;
        int dim;
    };
    const std::map<std::string, std::vector<Property>> schema = {
        {"xyzt", {{"xyz", CTICP_DTYPE_FLOAT64, 0, 3}, {"t", CTICP_DTYPE_FLOAT64, 24, 1}}},
        {"raw_point", {{"x", CTICP_DTYPE_FLOAT64, 0, 1}, {"y", CTICP_DTYPE_FLOAT64, 8, 1}, {"z", CTICP_DTYPE_FLOAT64, 16, 1}}},
        {"world_point",
         {{"x", CTICP_DTYPE_FLOAT64, 32, 1}, {"y", CTICP_DTYPE_FLOAT64, 40, 1}, {"z", CTICP_DTYPE_FLOAT64, 48, 1}}},
        {"properties",
         {{"raw_xyz", CTICP_DTYPE_FLOAT64, 0, 3}, {"t", CTICP_DTYPE_FLOAT64, 24, 1}, {"world_xyz", CTICP_DTYPE_FLOAT64, 32, 3},
          {"index_frame", CTICP_DTYPE_UINT32, 56, 1}}}};
    PLYSchemaMapper m;
    for (const auto &element : schema)
        for (const Property &p : element.second)
            for (int d = 0; d < p.dim; ++d)
                m.columns.push_back({element.first, p.dim == 1 ? p.name : std::string(p.name) + "_" + std::to_string(d),
                                     p.type, p.type, p.offset + 8 * (size_t) d});
    return m;
}

namespace detail {
inline std::string EncodePLY(const std::vector<PLYColumn> &columns, const void *records, size_t stride, size_t n,
                             int device) {
    std::vector<cticp_ply_property> props;
    for (const PLYColumn &c : columns)
        props.push_back({c.element.c_str(), c.name.c_str(), c.ply_dtype, c.src_dtype,
                         n ? static_cast<const char *>(records) + c.offset : nullptr, stride});
    const int64_t size = cticp_ply_write(device, props.data(), props.size(), n, nullptr, 0);
    if (size < 0) ct_icp::cticp_check((int) size);
    std::string out((size_t) size, '\0');
    const int64_t rc = cticp_ply_write(device, props.data(), props.size(), n, &out[0], out.size());
    if (rc < 0) ct_icp::cticp_check((int) rc);
    return out;
}
}  // namespace detail

// slam::WritePLY(os, points, schema); the default is WritePLY(os, points)'s mapper
inline void WritePLY(std::ostream &os, const std::vector<WPoint3D> &points,
                     const PLYSchemaMapper &schema = WPoint3DDefaultSchema(), int device = 0) {
    const std::string bytes = detail::EncodePLY(schema.columns, points.data(), sizeof(WPoint3D), points.size(), device);
    os.write(bytes.data(), (std::streamsize) bytes.size());
}
inline void WritePLY(const std::string &path, const std::vector<WPoint3D> &points,
                     const PLYSchemaMapper &schema = WPoint3DDefaultSchema(), int device = 0) {
    std::ofstream os(path, std::ios::out | std::ios::binary);
    WritePLY(os, points, schema, device);
}

// SavePosesAsPLY (io.cxx:320-351): element pose, qx qy qz qw x y z ref_t dest_t as double, ref_fid dest_fid as int
inline void SavePosesAsPLY(std::ostream &os, const std::vector<Pose> &poses, int device = 0) {
    std::vector<cticp_pose> raw(poses.size());
    for (size_t i = 0; i < poses.size(); ++i) {
        for (int k = 0; k < 4; ++k) raw[i].quat[k] = poses[i].pose.quat.c[k];
        for (int k = 0; k < 3; ++k) raw[i].tr[k] = poses[i].pose.tr.v[k];
        raw[i].ref_timestamp = poses[i].ref_timestamp;
        raw[i].dest_timestamp = poses[i].dest_timestamp;
        raw[i].ref_frame_id = poses[i].ref_frame_id;
        raw[i].dest_frame_id = poses[i].dest_frame_id;
    }
    const char *names[] = {"qx", "qy", "qz", "qw", "x", "y", "z", "ref_t", "dest_t"};
    std::vector<PLYColumn> columns;
    for (size_t k = 0; k < 9; ++k) columns.push_back({"pose", names[k], CTICP_DTYPE_FLOAT64, CTICP_DTYPE_FLOAT64, 8 * k});
    columns.push_back({"pose", "ref_fid", CTICP_DTYPE_INT32, CTICP_DTYPE_UINT32, offsetof(cticp_pose, ref_frame_id)});
    columns.push_back({"pose", "dest_fid", CTICP_DTYPE_INT32, CTICP_DTYPE_UINT32, offsetof(cticp_pose, dest_frame_id)});
    const std::string bytes = detail::EncodePLY(columns, raw.data(), sizeof(cticp_pose), raw.size(), device);
    os.write(bytes.data(), (std::streamsize) bytes.size());
}
inline void SavePosesAsPLY(const std::string &path, const std::vector<Pose> &poses, int device = 0) {
    std::ofstream os(path, std::ios::out | std::ios::binary);
    SavePosesAsPLY(os, poses, device);
}

// ReadPosesFromPLY (io.cxx:359-410), on the host
inline std::vector<Pose> ReadPosesFromPLY(std::istream &is) {
    const std::string bytes((std::istreambuf_iterator<char>(is)), std::istreambuf_iterator<char>());
    const int64_t n = cticp_ply_read_poses(bytes.data(), bytes.size(), nullptr, 0);
    if (n < 0) ct_icp::cticp_check((int) n);
    std::vector<cticp_pose> raw((size_t) n);
    if (n) cticp_ply_read_poses(bytes.data(), bytes.size(), raw.data(), raw.size());
    std::vector<Pose> out(raw.size());
    for (size_t i = 0; i < raw.size(); ++i) {
        for (int k = 0; k < 4; ++k) out[i].pose.quat.c[k] = raw[i].quat[k];
        for (int k = 0; k < 3; ++k) out[i].pose.tr.v[k] = raw[i].tr[k];
        out[i].ref_timestamp = raw[i].ref_timestamp;
        out[i].dest_timestamp = raw[i].dest_timestamp;
        out[i].ref_frame_id = raw[i].ref_frame_id;
        out[i].dest_frame_id = raw[i].dest_frame_id;
    }
    return out;
}
inline std::vector<Pose> ReadPosesFromPLY(const std::string &path) {
    std::ifstream is(path, std::ios::in | std::ios::binary);
    if (!is) throw ct_icp::CticpFailure(CTICP_ERR_INVALID_ARGUMENT, "cannot open " + path);
    return ReadPosesFromPLY(is);
}

}  // namespace slam

// ---- The reference's YAML readers (src/ct_icp/config.cpp, src/ct_icp/map.cpp:10-77, neighborhood_strategy.h:51-114) ---
// Templates over a node type with yaml-cpp's interface: `node[key]` (a node that converts to false when the key is
// absent), IsMap(), IsSequence(), `as<T>()` and range-for iteration. With YAML::Node they are the reference's own
// signatures, and the facade gains no dependency on yaml-cpp. Scalars convert through the node's `as<T>`; keys the
// option structs do not carry (output_*, log_to_file, the old map keys, ...) are converted and dropped. The Python
// readers (ct_icp_b200/config.py) are the same clauses; DESIGN.md §5.13 lists the quirks kept.
namespace ct_icp {

// ct_icp::SequenceOptions / DatasetOptions (include/ct_icp/dataset.h:270-293); `dataset` is DATASETEnumToString's
// name ("KITTI_raw", "NCLT", "SYNTHETIC", ...), empty when the node names none
struct SequenceOptions {
    std::string sequence_name;
    int start_frame_id = 0;
    int max_num_frames = -1;
};
struct DatasetOptions {
    std::string dataset;
    std::string root_path;
    bool fail_if_incomplete = false;
    double min_dist_lidar_center = 3.0;
    double max_dist_lidar_center = 100.0;
    int nclt_num_aggregated_pc = 220;
    bool use_all_datasets = true;
    std::vector<SequenceOptions> sequence_options;
};

namespace detail {
template <class T, class Node, class F>
inline void yaml_clause(const Node &node, const char *key, F &field) {   // OPTION_CLAUSE / FIND_OPTION
    if (node[key]) field = (F) node[key].template as<T>();
}
template <class Node>
inline void yaml_flag(const Node &node, const char *key, int32_t &field) {   // a bool clause into an int32 field
    if (node[key]) field = node[key].template as<bool>() ? 1 : 0;
}
template <class T, class Node>
inline void yaml_dropped(const Node &node, const char *key) {   // a clause into a field the structs do not carry
    if (node[key]) (void) node[key].template as<T>();
}
template <class Node>
inline bool yaml_enum(const Node &node, const char *key, std::string &out) {
    if (!node[key]) return false;
    out = node[key].template as<std::string>();
    return true;
}
inline int trunc_int(double x, const char *key) {   // the reference's double → int assignment (out of range refused)
    if (!(x > -2147483648.0 && x < 2147483648.0))
        throw std::runtime_error(std::string("`") + key + "` does not fit an int");
    return (int) x;
}
inline void check_enum(bool ok, const std::string &key, std::initializer_list<const char *> names, const std::string &got) {
    if (ok) return;
    std::string msg = "Check failed: ";
    bool first = true;
    for (const char *n : names) {
        msg += (first ? "" : " || ") + key + " == \"" + n + "\"";
        first = false;
    }
    throw std::runtime_error(msg + " (got " + got + ")");
}
}  // namespace detail

template <class Node>
CTICPOptions yaml_to_ct_icp_options(const Node &icp_node) {   // config.cpp:26-122
    using namespace detail;
    CTICPOptions o;
    yaml_clause<int>(icp_node, "threshold_voxel_occupancy", o.threshold_voxel_occupancy);
    yaml_clause<int>(icp_node, "num_iters_icp", o.num_iters_icp);
    yaml_clause<int>(icp_node, "min_number_neighbors", o.min_number_neighbors);
    yaml_clause<int>(icp_node, "max_number_neighbors", o.max_number_neighbors);
    yaml_clause<double>(icp_node, "max_dist_to_plane_ct_icp", o.max_dist_to_plane_ct_icp);
    yaml_clause<double>(icp_node, "threshold_orientation_norm", o.threshold_orientation_norm);
    yaml_clause<double>(icp_node, "threshold_translation_norm", o.threshold_translation_norm);
    yaml_flag(icp_node, "debug_print", o.debug_print);
    yaml_flag(icp_node, "point_to_plane_with_distortion", o.point_to_plane_with_distortion);
    yaml_clause<int>(icp_node, "num_closest_neighbors", o.num_closest_neighbors);
    yaml_clause<int>(icp_node, "ls_max_num_iters", o.ls_max_num_iters);
    yaml_clause<int>(icp_node, "ls_num_threads", o.ls_num_threads);
    yaml_clause<double>(icp_node, "ls_sigma", o.ls_sigma);
    yaml_clause<int>(icp_node, "min_num_residuals", o.min_num_residuals);
    yaml_clause<int>(icp_node, "max_num_residuals", o.max_num_residuals);
    yaml_clause<double>(icp_node, "weight_alpha", o.weight_alpha);
    yaml_clause<double>(icp_node, "weight_neighborhood", o.weight_neighborhood);
    yaml_clause<double>(icp_node, "ls_tolerant_min_threshold", o.ls_tolerant_min_threshold);
    yaml_clause<double>(icp_node, "power_planarity", o.power_planarity);
    yaml_flag(icp_node, "point_to_plane_with_distortion", o.point_to_plane_with_distortion);
    for (const char *k : {"output_normals", "output_lines", "output_weights", "output_residuals",
                          "output_neighborhood_info"})
        yaml_dropped<bool>(icp_node, k);
    yaml_clause<double>(icp_node, "threshold_linearity", o.threshold_linearity);
    yaml_clause<double>(icp_node, "threshold_planarity", o.threshold_planarity);
    yaml_clause<double>(icp_node, "weight_point_to_point", o.weight_point_to_point);
    yaml_clause<double>(icp_node, "outlier_distance", o.outlier_distance);
    yaml_flag(icp_node, "use_barycenter", o.use_barycenter);
    std::string s;
    if (yaml_enum(icp_node, "distance", s)) {
        if (s == "POINT_TO_PLANE") o.distance = CTICP_DIST_POINT_TO_PLANE;
        else if (s == "POINT_TO_LINE") o.distance = CTICP_DIST_POINT_TO_LINE;
        else if (s == "POINT_TO_POINT") o.distance = CTICP_DIST_POINT_TO_POINT;
        else if (s == "POINT_TO_DISTRIBUTION") o.distance = CTICP_DIST_POINT_TO_DISTRIBUTION;
        else throw std::runtime_error("Distance " + s + " not recognized as a valid distance");
    }
    if (yaml_enum(icp_node, "parametrization", s)) {
        if (s == "SIMPLE") o.parametrization = CTICP_PARAM_SIMPLE;
        else if (s == "CONTINUOUS_TIME") o.parametrization = CTICP_PARAM_CONTINUOUS_TIME;
        else throw std::runtime_error("Parametrization is not supported !");
    }
    if (yaml_enum(icp_node, "solver", s)) {
        if (s == "GN") o.solver = CTICP_SOLVER_GN;
        else if (s == "CERES") o.solver = CTICP_SOLVER_CERES;
        else if (s == "ROBUST") o.solver = CTICP_SOLVER_ROBUST;
        else throw std::runtime_error("Invalid Solver Options found: " + s + " Not in [GN, CERES, ROBUST]");
    }
    if (yaml_enum(icp_node, "loss_function", s)) {
        const char *names[] = {"STANDARD", "CAUCHY", "HUBER", "TOLERANT", "TRUNCATED"};
        int found = -1;
        for (int i = 0; i < 5; ++i)
            if (s == names[i]) found = i;
        if (found < 0) throw std::runtime_error("Unrecognised loss function " + s);
        o.loss_function = found;
    }
    return o;
}

template <class Node>
cticp_motion_model_options yaml_to_motion_model_options(const Node &node) {   // config.cpp:304-318
    using namespace detail;
    cticp_motion_model_options o = OdometryOptions().default_motion_model;
    yaml_clause<double>(node, "beta_location_consistency", o.beta_location_consistency);
    yaml_clause<double>(node, "beta_small_velocity", o.beta_small_velocity);
    yaml_clause<double>(node, "beta_orientation_consistency", o.beta_orientation_consistency);
    yaml_clause<double>(node, "beta_constant_velocity", o.beta_constant_velocity);
    yaml_clause<double>(node, "threshold_orientation_deg", o.threshold_orientation_deg);
    yaml_clause<double>(node, "threshold_translation_diff", o.threshold_translation_diff);
    yaml_flag(node, "log_if_invalid", o.log_if_invalid);
    std::string s;
    if (yaml_enum(node, "model", s)) {
        if (s == "CONSTANT_VELOCITY") o.model = CTICP_MM_CONSTANT_VELOCITY;
        else if (s == "SMALL_VELOCITY") o.model = CTICP_MM_SMALL_VELOCITY;
        else throw std::runtime_error("[ERROR] The option " + s +
                                      " is not a valid option. Valid options are: {CONSTANT_VELOCITY, SMALL_VELOCITY}");
    }
    return o;
}

// yaml_to_map_options (map.cpp:68-77): MULTI_RESOLUTION_VOXEL_HASHMAP, the old options without a map_type. The
// resolutions are sorted stably; the slots past the last one are zero; more than CTICP_MAX_RESOLUTIONS is refused.
template <class Node>
cticp_map_options yaml_to_map_options(const Node &node) {
    using namespace detail;
    cticp_map_options o;
    cticp_default_map_options(&o);
    if (!node["map_type"]) {   // old_map_options_from_yaml: one resolution (the default's first), one frame kept
        double size = o.resolutions[0].resolution, dmin = o.resolutions[0].min_distance_between_points;
        int npts = o.resolutions[0].max_num_points;
        yaml_clause<double>(node, "size_voxel_map", size);
        if (node["max_num_points_in_voxel"])
            npts = trunc_int(node["max_num_points_in_voxel"].template as<double>(), "max_num_points_in_voxel");
        yaml_clause<double>(node, "min_distance_points", dmin);
        cticp_legacy_map_options(&o, size, npts, dmin);
        return o;
    }
    if (node["map_type"].template as<std::string>() != "MULTI_RESOLUTION_VOXEL_HASHMAP")
        throw std::runtime_error("Not implemented error");
    if (node["resolutions"]) {
        const auto res = node["resolutions"];
        if (!res.IsSequence()) throw std::runtime_error("The node 'resolutions' in the yaml is not a sequence");
        std::vector<cticp_resolution_param> params;
        for (const auto &child : res) {
            if (!child.IsMap()) throw std::runtime_error("The following child node is not a Map");
            cticp_resolution_param p{};
            p.resolution = 0.5;   // ResolutionParam() (map.h:109-113)
            p.min_distance_between_points = 0.1;
            p.max_num_points = 40;
            yaml_clause<double>(child, "min_distance_between_points", p.min_distance_between_points);
            if (child["max_num_points"])
                p.max_num_points = trunc_int(child["max_num_points"].template as<double>(), "max_num_points");
            if (!child["resolution"]) throw std::runtime_error("Invalid Resolution Param in the yaml");
            p.resolution = child["resolution"].template as<double>();
            params.push_back(p);
        }
        if (params.empty()) throw std::runtime_error("The yaml does not define a valid set of resolutions for the map");
        if (params.size() > CTICP_MAX_RESOLUTIONS)
            throw std::runtime_error("the engine's map holds at most " + std::to_string(CTICP_MAX_RESOLUTIONS) +
                                     " resolutions");
        std::stable_sort(params.begin(), params.end(), [](const cticp_resolution_param &l,
                                                          const cticp_resolution_param &r) {
            return l.resolution < r.resolution;
        });
        o.num_resolutions = (int32_t) params.size();
        for (int i = 0; i < CTICP_MAX_RESOLUTIONS; ++i) o.resolutions[i] = i < (int) params.size() ? params[i]
                                                                                                  : cticp_resolution_param{};
    }
    yaml_clause<int>(node, "max_frames_to_keep", o.max_frames_to_keep);
    yaml_clause<double>(node, "default_radius", o.default_radius);
    return o;
}

// the neighborhood_strategy clause of yaml_to_odometry_options (config.cpp:155-168) and the strategies' FromYAML
template <class Node>
cticp_strategy_options yaml_to_strategy_options(const Node &node, const cticp_strategy_options &current) {
    using namespace detail;
    cticp_strategy_options o = current;
    std::string type = o.type == CTICP_STRATEGY_DISTANCE_BASED ? "DISTANCE_BASED_STRATEGY" : "NEAREST_NEIGHBOR_STRATEGY";
    yaml_enum(node, "type", type);
    if (type == "DISTANCE_BASED_STRATEGY")   // a fresh DistanceBasedStrategy::Options
        o = cticp_strategy_options{CTICP_STRATEGY_DISTANCE_BASED, 20, 8, 0, 60.0, 0.1, 2.0, 1.0};
    yaml_clause<int>(node, "max_num_neighbors", o.max_num_neighbors);
    yaml_clause<int>(node, "min_num_neighbors", o.min_num_neighbors);
    if (o.type == CTICP_STRATEGY_DISTANCE_BASED) {
        yaml_clause<double>(node, "distance_max", o.distance_max);
        yaml_clause<double>(node, "radius_min", o.radius_min);
        yaml_clause<double>(node, "radius_max", o.radius_max);
        yaml_clause<double>(node, "exponent", o.exponent);
    }
    return o;
}

template <class Node>
OdometryOptions yaml_to_odometry_options(const Node &odometry_node) {   // config.cpp:132-255
    using namespace detail;
    OdometryOptions o;
    yaml_clause<double>(odometry_node, "voxel_size", o.voxel_size);
    yaml_clause<double>(odometry_node, "max_distance", o.max_distance);
    yaml_clause<double>(odometry_node, "distance_error_threshold", o.distance_error_threshold);
    yaml_clause<double>(odometry_node, "orientation_error_threshold", o.orientation_error_threshold);
    yaml_clause<int>(odometry_node, "max_num_keypoints", o.max_num_keypoints);
    yaml_clause<double>(odometry_node, "sample_voxel_size", o.sample_voxel_size);
    o.map_options = odometry_node["map_options"] ? yaml_to_map_options(odometry_node["map_options"])
                                                 : yaml_to_map_options(odometry_node);
    if (odometry_node["neighborhood_strategy"])
        o.neighborhood_strategy = yaml_to_strategy_options(odometry_node["neighborhood_strategy"], o.neighborhood_strategy);
    yaml_dropped<double>(odometry_node, "min_distance_points");
    yaml_dropped<int>(odometry_node, "max_num_points_in_voxel");
    yaml_dropped<double>(odometry_node, "size_voxel_map");
    yaml_dropped<int>(odometry_node, "voxel_neighborhood");
    yaml_dropped<double>(odometry_node, "max_radius_neighborhood");
    yaml_clause<int>(odometry_node, "init_num_frames", o.init_num_frames);
    yaml_clause<double>(odometry_node, "init_voxel_size", o.init_voxel_size);
    yaml_clause<double>(odometry_node, "init_sample_voxel_size", o.init_sample_voxel_size);
    yaml_dropped<bool>(odometry_node, "log_to_file");
    yaml_dropped<std::string>(odometry_node, "log_file_destination");
    yaml_flag(odometry_node, "debug_print", o.debug_print);
    yaml_dropped<bool>(odometry_node, "debug_viz");
    yaml_flag(odometry_node, "do_no_insert", o.do_no_insert);
    yaml_flag(odometry_node, "always_insert", o.always_insert);
    yaml_clause<int>(odometry_node, "robust_minimal_level", o.robust_minimal_level);
    yaml_flag(odometry_node, "robust_registration", o.robust_registration);
    yaml_clause<double>(odometry_node, "robust_full_voxel_threshold", o.robust_full_voxel_threshold);
    yaml_flag(odometry_node, "robust_fail_early", o.robust_fail_early);
    yaml_clause<int>(odometry_node, "robust_num_attempts", o.robust_num_attempts);
    yaml_clause<int>(odometry_node, "robust_max_voxel_neighborhood", o.robust_max_voxel_neighborhood);
    yaml_clause<double>(odometry_node, "robust_threshold_relative_orientation", o.robust_threshold_relative_orientation);
    yaml_clause<double>(odometry_node, "robust_threshold_ego_orientation", o.robust_threshold_ego_orientation);
    if (odometry_node["default_motion_model"])
        o.default_motion_model = yaml_to_motion_model_options(odometry_node["default_motion_model"]);
    std::string s;
    if (yaml_enum(odometry_node, "motion_compensation", s)) {
        const bool ok = s == "NONE" || s == "CONSTANT_VELOCITY" || s == "ITERATIVE" || s == "CONTINUOUS";
        check_enum(ok, "motion_compensation", {"NONE", "CONSTANT_VELOCITY", "ITERATIVE", "CONTINUOUS"}, s);
        o.motion_compensation = s == "NONE" ? CTICP_MC_NONE : s == "CONSTANT_VELOCITY" ? CTICP_MC_CONSTANT_VELOCITY
                              : s == "ITERATIVE" ? CTICP_MC_ITERATIVE : CTICP_MC_CONTINUOUS;
    }
    if (yaml_enum(odometry_node, "sampling", s)) {
        check_enum(s == "GRID" || s == "ADAPTIVE" || s == "NONE", "sampling", {"GRID", "ADAPTIVE", "NONE"}, s);
        o.sampling = s == "NONE" ? CTICP_SAMPLING_NONE : s == "GRID" ? CTICP_SAMPLING_GRID : CTICP_SAMPLING_ADAPTIVE;
    }
    if (yaml_enum(odometry_node, "initialization", s)) {
        check_enum(s == "INIT_NONE" || s == "INIT_CONSTANT_VELOCITY", "initialization",
                   {"INIT_NONE", "INIT_CONSTANT_VELOCITY"}, s);
        o.initialization = s == "INIT_NONE" ? CTICP_INIT_NONE : CTICP_INIT_CONSTANT_VELOCITY;
    }
    if (odometry_node["ct_icp_options"]) {
        const CTICPOptions icp = yaml_to_ct_icp_options(odometry_node["ct_icp_options"]);
        o.ct_icp_options = icp;
    }
    return o;
}

template <class Node>
DatasetOptions yaml_to_dataset_options(const Node &dataset_node) {   // config.cpp:264-291
    using namespace detail;
    DatasetOptions o;
    if (dataset_node["dataset"]) {   // DATASETFromString: case-insensitive, hilti is HILTI_2021
        const std::string name = dataset_node["dataset"].template as<std::string>();
        std::string lc = name;
        std::transform(lc.begin(), lc.end(), lc.begin(), [](unsigned char c) { return (char) std::tolower(c); });
        const std::map<std::string, std::string> names = {
            {"kitti_carla", "KITTI_CARLA"}, {"kitti_360", "KITTI_360"}, {"kitti", "KITTI"}, {"hilti", "HILTI_2021"},
            {"hilti_2021", "HILTI_2021"}, {"hilti_2022", "HILTI_2022"}, {"kitti_raw", "KITTI_raw"}, {"nclt", "NCLT"},
            {"synthetic", "SYNTHETIC"}, {"ply_directory", "PLY_DIRECTORY"}};
        auto it = names.find(lc);
        if (it == names.end()) throw std::runtime_error("The `dataset` name: " + name + " is invalid.");
        o.dataset = it->second;
    }
    yaml_clause<std::string>(dataset_node, "root_path", o.root_path);
    yaml_clause<bool>(dataset_node, "fail_if_incomplete", o.fail_if_incomplete);
    yaml_clause<float>(dataset_node, "min_dist_lidar_center", o.min_dist_lidar_center);
    yaml_clause<int>(dataset_node, "nclt_num_aggregated_pc", o.nclt_num_aggregated_pc);
    yaml_clause<float>(dataset_node, "max_dist_lidar_center", o.max_dist_lidar_center);
    yaml_clause<bool>(dataset_node, "use_all_datasets", o.use_all_datasets);
    if (dataset_node["sequence_options"]) {
        o.sequence_options.clear();
        for (const auto &seq_node : dataset_node["sequence_options"]) {
            SequenceOptions s;
            yaml_clause<std::string>(seq_node, "sequence_name", s.sequence_name);
            yaml_clause<int>(seq_node, "start_frame_id", s.start_frame_id);
            yaml_clause<int>(seq_node, "max_num_frames", s.max_num_frames);
            o.sequence_options.push_back(s);
        }
    }
    return o;
}

template <class Node>
std::vector<DatasetOptions> yaml_to_dataset_options_vector(const Node &node) {   // config.cpp:294-301
    std::vector<DatasetOptions> out;
    for (const auto &child : node) out.push_back(yaml_to_dataset_options(child));
    return out;
}

}  // namespace ct_icp
