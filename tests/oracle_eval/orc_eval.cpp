// ORACLE — TEST INFRASTRUCTURE ONLY. The scoring entry points of include/cticp.h (cticp_kitti_evaluate,
// cticp_trajectory_metrics, cticp_trajectory_distances), prefixed orc_, over orc_eval.h: the tests drive the engine and
// this restatement through the same Python binding. Host memory only; estimates are scored one after the other.
// Built by __graft_entry__.build() and by tests/oracle_eval_lib.py into liborc_eval.so.
#include <cstring>
#include <string>
#include <vector>

#include "../../include/cticp.h"
#include "orc_eval.h"

namespace {
thread_local std::string g_last_error;

template <typename F>
int64_t Guard(F &&f) {
    try {
        return f();
    } catch (const std::invalid_argument &e) {
        g_last_error = e.what();
        return CTICP_ERR_INVALID_ARGUMENT;
    } catch (const std::exception &e) {
        g_last_error = e.what();
        return CTICP_ERR_INTERNAL;
    }
}

std::vector<orc::Pose> FromC(const cticp_pose *c, size_t n) {
    std::vector<orc::Pose> v(n);
    for (size_t i = 0; i < n; ++i) {
        v[i].pose.quat = orc::Quat(c[i].quat[0], c[i].quat[1], c[i].quat[2], c[i].quat[3]);   // as given
        v[i].pose.tr = orc::Vec3(c[i].tr[0], c[i].tr[1], c[i].tr[2]);
        v[i].ref_timestamp = c[i].ref_timestamp;
        v[i].dest_timestamp = c[i].dest_timestamp;
        v[i].ref_frame_id = c[i].ref_frame_id;
        v[i].dest_frame_id = c[i].dest_frame_id;
    }
    return v;
}
void Store(const orc::SE3 &T, double quat[4], double tr[3]) {
    quat[0] = T.quat.x; quat[1] = T.quat.y; quat[2] = T.quat.z; quat[3] = T.quat.w;
    tr[0] = T.tr.x; tr[1] = T.tr.y; tr[2] = T.tr.z;
}
}  // namespace

extern "C" {

const char *orc_last_error(void) { return g_last_error.c_str(); }

int64_t orc_kitti_evaluate(int device, const cticp_pose *gt, size_t n, const cticp_pose *est, size_t num_estimates,
                           const double *lengths, size_t num_lengths, cticp_kitti_errors *out, double *tab_errors,
                           size_t cap) {
    (void) device;
    return Guard([&] {
        if (!gt || !est || !out || !num_estimates) throw std::invalid_argument("bad argument");
        const std::vector<orc::Pose> g = FromC(gt, n);
        const std::vector<double> lens(lengths, lengths + num_lengths);
        int64_t count = 0;
        for (size_t b = 0; b < num_estimates; ++b) {
            const orc::eval::KittiErrors e = orc::eval::EvaluatePoses(g, FromC(est + b * n, n), lens);
            out[b] = cticp_kitti_errors{e.mean_rpe, e.mean_ape, e.max_ape, e.mean_local_err, e.max_local_err,
                                        e.index_max_local_err};
            count = (int64_t) e.tab_errors.size();
            for (size_t k = 0; k < e.tab_errors.size() && k < cap && tab_errors; ++k) {
                tab_errors[2 * (b * cap + k)] = e.tab_errors[k].first;
                tab_errors[2 * (b * cap + k) + 1] = e.tab_errors[k].second;
            }
        }
        return count;
    });
}

int64_t orc_trajectory_metrics(int device, const cticp_pose *gt, size_t n, const cticp_pose *est, size_t num_estimates,
                               double segment_length, cticp_traj_metrics *out, cticp_traj_segment *segments,
                               size_t cap) {
    (void) device;
    return Guard([&] {
        if (!gt || !est || !out || !num_estimates) throw std::invalid_argument("bad argument");
        const std::vector<orc::Pose> g = FromC(gt, n);
        int64_t count = 0;
        for (size_t b = 0; b < num_estimates; ++b) {
            const orc::eval::Metrics m = orc::eval::ComputeTrajectoryMetrics(g, FromC(est + b * n, n), segment_length);
            cticp_traj_metrics &r = out[b];
            r.total_distance = m.total_distance;
            r.mean_ate = m.mean_ate;
            r.max_ate = m.max_ate;
            r.max_ate_idx = m.max_ate_idx;
            r.segment_mean_ate = m.segment_mean_ate;
            r.segment_mean_ate_ratio = m.segment_mean_ate_ratio;
            r.num_segments = (int64_t) m.segments.size();
            Store(m.rigid_transform, r.quat, r.tr);
            count = (int64_t) m.segments.size();
            for (size_t k = 0; k < m.segments.size() && k < cap && segments; ++k) {
                const orc::eval::Segment &s = m.segments[k];
                cticp_traj_segment &o = segments[b * cap + k];
                o.segment_length = s.segment_length;
                o.start_idx = s.start_idx;
                o.end_idx = s.end_idx;
                o.loc_error = s.loc_error;
                Store(s.rigid_transform, o.quat, o.tr);
            }
        }
        return count;
    });
}

int orc_trajectory_distances(int device, const cticp_pose *gt, size_t n, int kind, double *out) {
    (void) device;
    return (int) Guard([&] {
        if (!gt || !out || n == 0 || (kind != 0 && kind != 1)) throw std::invalid_argument("bad argument");
        const std::vector<orc::Pose> g = FromC(gt, n);
        const std::vector<double> d = kind == 0 ? orc::eval::KittiDistances(g) : orc::eval::MetricsDistances(g);
        memcpy(out, d.data(), sizeof(double) * n);
        return (int64_t) 0;
    });
}

// test tap: the 3×3 SVD of the oracle (row-major A, U, V)
void orc_svd3(const double *a, double *u, double *v) {
    orc::Mat3 A, U, V;
    for (int i = 0; i < 9; ++i) A(i / 3, i % 3) = a[i];
    orc::eval::SVD3(A, U, V);
    for (int i = 0; i < 9; ++i) {
        u[i] = U(i / 3, i % 3);
        v[i] = V(i / 3, i % 3);
    }
}

}  // extern "C"
