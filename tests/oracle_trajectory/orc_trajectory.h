// ORACLE — TEST INFRASTRUCTURE ONLY. Not linked into, imported by, or shipped with the product (ct_icp_b200/).
//
// orc_trajectory.h — slam::LinearContinuousTrajectory restated in the oracle's fp64 types (orc_math.h), written from the
// reference's behaviour: src/SlamCore/trajectory.cxx (DoInterpolatePose :16-30, GetClosestPosesIds :54-140,
// TransformPoint :143-155, Create / CheckConsistency :164-206) and include/SlamCore/types.h (GetAlphaTimestamp
// :192-219, TSE3 :353-366, InterpolatePoseAlpha :434-452). Every step is plain host fp64 with libm, one point at a time.
// The reference's CHECK failures are std::invalid_argument here.
#pragma once
#include <algorithm>
#include <cmath>
#include <limits>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../oracle/orc_math.h"

namespace orc {

class LinearContinuousTrajectory {
public:
    // Create(poses, check_consistency = true); equal keys keep their input order (stable sort). A NaN dest_timestamp is
    // refused: std::sort's order is undefined on it.
    static LinearContinuousTrajectory Create(std::vector<Pose> poses) {
        if (poses.empty()) throw std::invalid_argument("The trajectory created is invalid");
        for (const Pose &p : poses)
            if (std::isnan(p.dest_timestamp)) throw std::invalid_argument("NaN dest_timestamp");
        std::stable_sort(poses.begin(), poses.end(), [](const Pose &l, const Pose &r) {
            return l.dest_frame_id < r.dest_frame_id ||
                   (l.dest_frame_id == r.dest_frame_id && l.dest_timestamp < r.dest_timestamp);
        });
        LinearContinuousTrajectory r;
        r.reference_frame_ = poses.front().ref_frame_id;
        r.min_ts_ = std::numeric_limits<double>::max();
        r.max_ts_ = std::numeric_limits<double>::min();   // sic: the smallest positive double
        for (const Pose &p : poses) {
            if (p.dest_timestamp < r.min_ts_) r.min_ts_ = p.dest_timestamp;
            if (p.dest_timestamp > r.max_ts_) r.max_ts_ = p.dest_timestamp;
        }
        r.poses_ = std::move(poses);
        r.CheckConsistency();
        return r;
    }

    const std::vector<Pose> &Poses() const { return poses_; }
    double MinTimestamp() const { return min_ts_; }
    double MaxTimestamp() const { return max_ts_; }

    // the bounds check (:54-75, clip_on_bounds = true): true when it decided the indices
    bool Clip(double t, size_t &lo, size_t &up) const {
        if (MinTimestamp() >= t && t >= MaxTimestamp()) {
            if (t <= MinTimestamp()) lo = up = 0;
            else lo = up = poses_.size() - 1;
            return true;
        }
        return false;
    }
    void GetClosestPosesIds(double t, size_t &lo, size_t &up) const {   // :78-108
        if (Clip(t, lo, up)) return;
        auto it = std::lower_bound(poses_.begin(), poses_.end(), t,
                                   [](const Pose &p, double ts) { return p.dest_timestamp < ts; });
        up = (size_t) std::distance(poses_.begin(), it);
        if (up >= poses_.size()) {
            up = lo = poses_.size() - 1;
            return;
        }
        lo = up;
        double below = poses_[lo].dest_timestamp;
        while (below > t) {
            if (lo <= 0) break;
            lo--;
            below = poses_[lo].dest_timestamp;
        }
    }
    void GetClosestPosesIds(double t, uint32_t frame_id, size_t &lo, size_t &up) const {   // :111-140
        if (Clip(t, lo, up)) return;
        auto it = std::lower_bound(poses_.begin(), poses_.end(), std::make_pair(frame_id, t),
                                   [](const Pose &p, std::pair<uint32_t, double> k) {
                                       return p.dest_frame_id < k.first ||
                                              (p.dest_frame_id == k.first && p.dest_timestamp < k.second);
                                   });
        if (it == poses_.end()) {
            if (poses_.back().dest_frame_id == frame_id) {
                lo = up = poses_.size() - 1;
                return;
            }
            throw std::invalid_argument("Invalid frame or trajectory. Got request for " + std::to_string(frame_id) +
                                        " when max frame_id in trajectory is " +
                                        std::to_string(poses_.back().dest_frame_id));
        }
        up = (size_t) std::distance(poses_.begin(), it);
        lo = up == 0 ? 0 : up - 1;
    }
    Pose DoInterpolatePose(double t, size_t lo, size_t up) const {   // :16-30
        const Pose &p0 = poses_[lo];
        if (lo == up) return p0;
        const Pose &p1 = poses_[up];
        return p0.InterpolatePoseAlpha(p1, p0.GetAlphaTimestamp(t, p1));
    }
    Pose InterpolatePose(double t) const {
        size_t lo = 0, up = 0;
        GetClosestPosesIds(t, lo, up);
        return DoInterpolatePose(t, lo, up);
    }
    Pose InterpolatePoseWithFrameId(double t, uint32_t frame_id) const {
        size_t lo = 0, up = 0;
        GetClosestPosesIds(t, frame_id, lo, up);
        return DoInterpolatePose(t, lo, up);
    }
    Vec3 TransformPoint(const Vec3 &raw, double t) const { return InterpolatePose(t).pose * raw; }
    Vec3 TransformPoint(const Vec3 &raw, double t, uint32_t frame_id) const {
        return InterpolatePoseWithFrameId(t, frame_id).pose * raw;
    }

private:
    void CheckConsistency() const {   // :189-206
        uint32_t previous_frame = poses_.front().dest_frame_id;
        double previous_ts = poses_.front().dest_timestamp;
        for (size_t i = 1; i < poses_.size(); ++i) {
            const Pose &p = poses_[i];
            if (p.ref_frame_id != reference_frame_) throw std::invalid_argument("Inconsistent reference frames");
            if (p.dest_frame_id != previous_frame && !(p.dest_timestamp >= previous_ts))
                throw std::invalid_argument("Inconsistent Timestamps");
            previous_frame = p.dest_frame_id;
            previous_ts = p.dest_timestamp;
        }
    }

    std::vector<Pose> poses_;
    double min_ts_ = 0, max_ts_ = 0;
    uint32_t reference_frame_ = 0;
};

}  // namespace orc
