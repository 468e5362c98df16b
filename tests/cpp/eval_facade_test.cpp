// slam::kitti::EvaluatePoses and slam::ComputeTrajectoryMetrics of the C++ facade (ct_icp_b200/odometry.hpp) against the
// CPU restatement of the reference (tests/oracle_eval/orc_eval.h) on a seeded odometry-shaped trajectory: the pose-list
// forms, the LinearContinuousTrajectory form, the distances, the segments and a refused size mismatch.
// Exit 0 and "EVAL FACADE OK" on success; exit 42 when no device is usable (CTICP_ERR_NO_DEVICE); 1 on a mismatch.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "ct_icp_b200/odometry.hpp"
#include "orc_eval.h"
#include "orc_trajectory.h"

namespace {
int failures = 0;
void expect(bool ok, const char *what, double a = 0, double b = 0) {
    if (!ok) {
        std::printf("MISMATCH %s: %.17g vs %.17g\n", what, a, b);
        ++failures;
    }
}
orc::Pose ToOracle(const slam::Pose &p) {
    orc::Pose o;
    o.pose.quat = orc::Quat(p.pose.quat.c[0], p.pose.quat.c[1], p.pose.quat.c[2], p.pose.quat.c[3]);
    o.pose.tr = orc::Vec3(p.pose.tr[0], p.pose.tr[1], p.pose.tr[2]);
    o.dest_timestamp = p.dest_timestamp;
    o.dest_frame_id = p.dest_frame_id;
    return o;
}
std::vector<orc::Pose> ToOracle(const std::vector<slam::Pose> &v) {
    std::vector<orc::Pose> o;
    for (const auto &p : v) o.push_back(ToOracle(p));
    return o;
}
bool close(double a, double b, double tol) { return std::fabs(a - b) <= tol || (std::isnan(a) && std::isnan(b)); }
void CompareKitti(const slam::kitti::seq_errors &a, const orc::eval::KittiErrors &b) {
    expect(a.tab_errors.size() == b.tab_errors.size(), "pair count", a.tab_errors.size(), b.tab_errors.size());
    for (size_t k = 0; k < a.tab_errors.size() && k < b.tab_errors.size(); ++k) {
        expect(close(a.tab_errors[k].t_err, b.tab_errors[k].first, 1e-11), "t_err", a.tab_errors[k].t_err, b.tab_errors[k].first);
        // 3e-8 rad before the division by the shortest length of these runs (7.5 m): acos near 1 amplifies rounding
        expect(close(a.tab_errors[k].r_err, b.tab_errors[k].second, 4e-9), "r_err", a.tab_errors[k].r_err, b.tab_errors[k].second);
    }
    expect(close(a.mean_rpe, b.mean_rpe, 1e-10), "mean_rpe", a.mean_rpe, b.mean_rpe);
    expect(close(a.mean_ape, b.mean_ape, 1e-10), "mean_ape", a.mean_ape, b.mean_ape);
    expect(close(a.max_ape, b.max_ape, 1e-10), "max_ape", a.max_ape, b.max_ape);
    expect(close(a.mean_local_err, b.mean_local_err, 1e-10), "mean_local_err", a.mean_local_err, b.mean_local_err);
    expect(close(a.max_local_err, b.max_local_err, 1e-10), "max_local_err", a.max_local_err, b.max_local_err);
    expect(a.index_max_local_err == b.index_max_local_err, "index_max_local_err", a.index_max_local_err,
           (double) b.index_max_local_err);
}
}  // namespace

int main() {
    std::mt19937_64 rng(20261017);
    std::normal_distribution<double> nd(0.0, 1.0);
    // 1500 poses along a drifting heading, ~0.8 m apart; the estimate is the ground truth with noise
    std::vector<slam::Pose> gt, est;
    double yaw = 0, x = 0, y = 0;
    for (int i = 0; i < 1500; ++i) {
        yaw += 0.02 * nd(rng);
        slam::Pose p;
        p.pose.quat.c[2] = std::sin(yaw / 2);
        p.pose.quat.c[3] = std::cos(yaw / 2);
        p.pose.tr[0] = x;
        p.pose.tr[1] = y;
        p.pose.tr[2] = 0.01 * nd(rng);
        p.dest_timestamp = 0.1 * i;
        p.dest_frame_id = (slam::frame_id_t) i;
        gt.push_back(p);
        slam::Pose e = p;
        double n = 0;
        for (int c = 0; c < 4; ++c) n += (e.pose.quat.c[c] += 0.003 * nd(rng)) * e.pose.quat.c[c];
        for (int c = 0; c < 4; ++c) e.pose.quat.c[c] /= std::sqrt(n);
        for (int c = 0; c < 3; ++c) e.pose.tr[c] += 0.2 * nd(rng);
        est.push_back(e);
        x += 0.8 * std::cos(yaw);
        y += 0.8 * std::sin(yaw);
    }
    const std::vector<orc::Pose> ogt = ToOracle(gt), oest = ToOracle(est);

    slam::kitti::seq_errors driving;
    try {
        driving = slam::kitti::EvaluatePoses(gt, est);
    } catch (const ct_icp::CticpFailure &e) {
        std::printf("%s\n", e.what());
        return e.code == CTICP_ERR_NO_DEVICE ? 42 : 1;
    }
    CompareKitti(driving, orc::eval::EvaluatePoses(ogt, oest, slam::kitti::kitti_segment_lengths));
    CompareKitti(slam::kitti::EvaluatePoses(gt, est, false),
                 orc::eval::EvaluatePoses(ogt, oest, slam::kitti::indoor_segment_lengths));
    const std::vector<double> custom{7.5, 33.0};
    CompareKitti(slam::kitti::EvaluatePoses(gt, est, custom), orc::eval::EvaluatePoses(ogt, oest, custom));

    // the trajectory form: the estimate's frames as begin / end poses, looked up at the ground truth's timestamps
    std::vector<slam::Pose> frames;
    for (size_t i = 0; i + 1 < est.size(); i += 2) {
        slam::Pose b = est[i], e = est[i + 1];
        b.dest_timestamp += 0.02;
        e.dest_timestamp += 0.02;
        b.dest_frame_id = e.dest_frame_id = (slam::frame_id_t) (i / 2);
        frames.push_back(b);
        frames.push_back(e);
    }
    const auto otraj = orc::LinearContinuousTrajectory::Create(ToOracle(frames));
    std::vector<orc::Pose> ointerp;
    for (const auto &p : ogt) ointerp.push_back(otraj.InterpolatePose(p.dest_timestamp));
    const slam::LinearContinuousTrajectory traj = slam::LinearContinuousTrajectory::Create(std::move(frames));
    CompareKitti(slam::kitti::EvaluatePoses(gt, traj), orc::eval::EvaluatePoses(ogt, ointerp, slam::kitti::kitti_segment_lengths));

    // ComputeTrajectoryMetrics
    const slam::metrics_t m = slam::ComputeTrajectoryMetrics(gt, est, 10.0);
    const orc::eval::Metrics om = orc::eval::ComputeTrajectoryMetrics(ogt, oest, 10.0);
    expect(m.distances.size() == om.distances.size(), "distances size");
    for (size_t i = 0; i < m.distances.size() && i < om.distances.size(); ++i)
        expect(m.distances[i] == om.distances[i], "distances (bit for bit)", m.distances[i], om.distances[i]);
    expect(m.total_distance == om.total_distance, "total_distance", m.total_distance, om.total_distance);
    expect(close(m.mean_ate, om.mean_ate, 1e-10), "mean_ate", m.mean_ate, om.mean_ate);
    expect(close(m.max_ate, om.max_ate, 1e-10), "max_ate", m.max_ate, om.max_ate);
    expect((int64_t) m.max_ate_idx == om.max_ate_idx, "max_ate_idx", (double) m.max_ate_idx, (double) om.max_ate_idx);
    expect(close(m.segment_mean_ate, om.segment_mean_ate, 1e-10), "segment_mean_ate", m.segment_mean_ate, om.segment_mean_ate);
    expect(close(m.segment_mean_ate_ratio, om.segment_mean_ate_ratio, 1e-10), "segment_mean_ate_ratio",
           m.segment_mean_ate_ratio, om.segment_mean_ate_ratio);
    expect(m.trajectory_segments.size() == om.segments.size() && m.loc_errors.size() == om.segments.size(), "segments",
           m.trajectory_segments.size(), om.segments.size());
    for (size_t k = 0; k < m.trajectory_segments.size() && k < om.segments.size(); ++k) {
        expect(m.trajectory_segments[k].start_idx == (size_t) om.segments[k].start_idx &&
                   m.trajectory_segments[k].end_idx == (size_t) om.segments[k].end_idx,
               "segment bounds");
        expect(m.trajectory_segments[k].segment_length == om.segments[k].segment_length, "segment_length");
        expect(close(m.loc_errors[k], om.segments[k].loc_error, 1e-10), "loc_error", m.loc_errors[k], om.segments[k].loc_error);
        expect(m.trajectory_segments[k].rigid_transform.has_value(), "segment transform");
    }
    expect(m.rigid_transform.has_value(), "rigid_transform");

    std::vector<slam::Pose> shorter(est.begin(), est.end() - 1);
    try {
        slam::kitti::EvaluatePoses(gt, shorter);
        expect(false, "a size mismatch was accepted");
    } catch (const ct_icp::CticpFailure &e) {
        expect(e.code == CTICP_ERR_INVALID_ARGUMENT, "error code", e.code, CTICP_ERR_INVALID_ARGUMENT);
    }
    if (failures) {
        std::printf("%d mismatches\n", failures);
        return 1;
    }
    std::printf("EVAL FACADE OK (%zu poses, %zu pairs, %zu segments)\n", gt.size(), driving.tab_errors.size(),
                m.trajectory_segments.size());
    return 0;
}
