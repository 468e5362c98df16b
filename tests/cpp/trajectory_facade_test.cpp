// slam::LinearContinuousTrajectory of the C++ facade (ct_icp_b200/odometry.hpp) against the CPU restatement of the
// reference (tests/oracle_trajectory/orc_trajectory.h): Create → Poses / MinTimestamp / MaxTimestamp, InterpolatePose,
// InterpolatePoseWithFrameId, TransformPoint and RawPointsToWorldPoints on a seeded odometry-shaped trajectory.
// Exit 0 and "TRAJECTORY FACADE OK" on success; exit 42 when no device is usable (CTICP_ERR_NO_DEVICE); 1 on a mismatch.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "ct_icp_b200/odometry.hpp"
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
    o.ref_timestamp = p.ref_timestamp;
    o.dest_timestamp = p.dest_timestamp;
    o.ref_frame_id = p.ref_frame_id;
    o.dest_frame_id = p.dest_frame_id;
    return o;
}
void ComparePose(const slam::Pose &a, const orc::Pose &b) {
    const double qb[4] = {b.pose.quat.x, b.pose.quat.y, b.pose.quat.z, b.pose.quat.w};
    // (a NaN timestamp looked up by frame id interpolates with a NaN alpha on both sides)
    auto close = [](double x, double y, double tol) { return std::fabs(x - y) <= tol || (std::isnan(x) && std::isnan(y)); };
    for (int k = 0; k < 4; ++k) expect(close(a.pose.quat.c[k], qb[k], 1e-14), "quat", a.pose.quat.c[k], qb[k]);
    for (int k = 0; k < 3; ++k) expect(close(a.pose.tr[k], b.pose.tr[k], 1e-12), "tr", a.pose.tr[k], b.pose.tr[k]);
    expect(a.dest_timestamp == b.dest_timestamp || (std::isnan(a.dest_timestamp) && std::isnan(b.dest_timestamp)),
           "dest_timestamp", a.dest_timestamp, b.dest_timestamp);
    expect(a.dest_frame_id == b.dest_frame_id, "dest_frame_id", a.dest_frame_id, b.dest_frame_id);
    expect(a.ref_frame_id == b.ref_frame_id && a.ref_timestamp == b.ref_timestamp, "ref_*");
}
}  // namespace

int main() {
    std::mt19937_64 rng(20261017);
    std::normal_distribution<double> nd(0.0, 1.0);
    std::uniform_real_distribution<double> ud(0.0, 1.0);
    // 12 frames of begin / end poses, small motion, every other boundary shared with the next frame's begin
    std::vector<slam::Pose> poses;
    double q[4] = {0, 0, 0, 1}, tr[3] = {0, 0, 0}, t = 50.0;
    for (int k = 0; k < 12; ++k) {
        for (int e = 0; e < 2; ++e) {
            slam::Pose p;
            double n = 0;
            for (int c = 0; c < 4; ++c) { q[c] += 0.02 * nd(rng); n += q[c] * q[c]; }
            for (int c = 0; c < 4; ++c) p.pose.quat.c[c] = q[c] / std::sqrt(n);
            for (int c = 0; c < 3; ++c) p.pose.tr[c] = tr[c] += nd(rng);
            p.dest_timestamp = t + 0.1 * e;
            p.dest_frame_id = (slam::frame_id_t) k;
            p.ref_frame_id = 0;
            poses.push_back(p);
        }
        t += (k % 2) ? 0.1 : 0.105;
    }
    std::vector<orc::Pose> oposes;
    for (auto &p : poses) oposes.push_back(ToOracle(p));
    std::vector<slam::Pose> shuffled(poses.rbegin(), poses.rend());
    slam::LinearContinuousTrajectory traj = [&] {
        try {
            return slam::LinearContinuousTrajectory::Create(std::move(shuffled));
        } catch (const ct_icp::CticpFailure &e) {
            std::printf("%s\n", e.what());
            std::exit(e.code == CTICP_ERR_NO_DEVICE ? 42 : 1);
        }
    }();
    const auto oracle = orc::LinearContinuousTrajectory::Create(oposes);
    expect(traj.Poses().size() == oracle.Poses().size(), "size");
    for (size_t i = 0; i < traj.Poses().size(); ++i) ComparePose(traj.Poses()[i], oracle.Poses()[i]);
    expect(traj.MinTimestamp() == oracle.MinTimestamp(), "MinTimestamp", traj.MinTimestamp(), oracle.MinTimestamp());
    expect(traj.MaxTimestamp() == oracle.MaxTimestamp(), "MaxTimestamp", traj.MaxTimestamp(), oracle.MaxTimestamp());

    const double lo = oracle.MinTimestamp() - 0.2, hi = oracle.MaxTimestamp() + 0.2;
    for (int i = 0; i < 300; ++i) {
        const double ts = i == 0 ? NAN : lo + (hi - lo) * ud(rng);
        const int fid = (int) (ud(rng) * 12);
        ComparePose(traj.InterpolatePose(ts), oracle.InterpolatePose(ts));
        ComparePose(traj.InterpolatePoseWithFrameId(ts, fid), oracle.InterpolatePoseWithFrameId(ts, (uint32_t) fid));
        slam::Vec3d raw;
        for (int c = 0; c < 3; ++c) raw[c] = 60.0 * (ud(rng) - 0.5);
        const orc::Vec3 oraw(raw[0], raw[1], raw[2]);
        const slam::Vec3d w = traj.TransformPoint(raw, ts), wf = traj.TransformPoint(raw, ts, fid);
        const orc::Vec3 ow = oracle.TransformPoint(oraw, ts), owf = oracle.TransformPoint(oraw, ts, (uint32_t) fid);
        for (int c = 0; c < 3; ++c) {
            expect(std::fabs(w[c] - ow[c]) <= 1e-10 || (std::isnan(w[c]) && std::isnan(ow[c])), "TransformPoint", w[c], ow[c]);
            expect(std::fabs(wf[c] - owf[c]) <= 1e-10 || (std::isnan(wf[c]) && std::isnan(owf[c])), "TransformPoint(fid)",
                   wf[c], owf[c]);
        }
    }

    // RawPointsToWorldPoints: 12 scans of 2000 points concatenated, each frame's points inside its own sweep
    std::vector<slam::WPoint3D> points;
    for (int k = 0; k < 12; ++k) {
        const double b = oracle.Poses()[2 * k].dest_timestamp, e = oracle.Poses()[2 * k + 1].dest_timestamp;
        for (int i = 0; i < 2000; ++i) {
            slam::WPoint3D p;
            for (int c = 0; c < 3; ++c) p.RawPoint()[c] = 100.0 * (ud(rng) - 0.5);
            p.Timestamp() = b + (e - b) * ud(rng);
            p.index_frame = (slam::frame_id_t) k;
            points.push_back(p);
        }
    }
    const std::vector<slam::WPoint3D> before = points;
    slam::RawPointsToWorldPoints(points, traj);
    for (size_t i = 0; i < points.size(); ++i) {
        const auto &p = points[i];
        expect(p.Timestamp() == before[i].Timestamp() && p.index_frame == before[i].index_frame &&
                   p.RawPoint()[0] == before[i].RawPoint()[0], "raw fields kept");
        const orc::Vec3 ow = oracle.TransformPoint(orc::Vec3(p.RawPoint()[0], p.RawPoint()[1], p.RawPoint()[2]), p.Timestamp(),
                                                   p.index_frame);
        for (int c = 0; c < 3; ++c)
            expect(std::fabs(p.WorldPoint()[c] - ow[c]) <= 1e-10, "RawPointsToWorldPoints", p.WorldPoint()[c], ow[c]);
    }

    // CheckConsistency: a timestamp that decreases where the frame id changes
    std::vector<slam::Pose> bad = {poses[0], poses[2]};
    bad[1].dest_timestamp = bad[0].dest_timestamp - 1.0;
    try {
        slam::LinearContinuousTrajectory::Create(std::move(bad));
        expect(false, "inconsistent trajectory accepted");
    } catch (const ct_icp::CticpFailure &e) {
        expect(e.code == CTICP_ERR_INVALID_ARGUMENT, "error code", e.code, CTICP_ERR_INVALID_ARGUMENT);
    }
    if (failures) {
        std::printf("%d mismatches\n", failures);
        return 1;
    }
    std::printf("TRAJECTORY FACADE OK (%zu poses, %zu points)\n", traj.Poses().size(), points.size());
    return 0;
}
