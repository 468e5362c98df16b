// ORACLE — TEST INFRASTRUCTURE ONLY. Not linked into, imported by, or shipped with the product (ct_icp_b200/).
//
// orc_eval.h — kitti::EvaluatePoses and ComputeTrajectoryMetrics restated in the oracle's fp64 types (orc_math.h), one
// pose at a time, written from the reference's behaviour: src/SlamCore/eval.cxx (ComputeMeanRPE :35-76, EvaluatePoses
// :136-178, ComputeTrajectoryMetrics :184-291), src/SlamCore/geometry.cxx:7-46 (OrthogonalProcrustes) and
// include/SlamCore/types.h:326-350, 474-479. Sums run sequentially in index order, as the reference's loops do.
// Deviations, as in the engine: the segment ratio's accumulator starts at 0 (the reference leaves it uninitialised), and
// Eigen's general 4×4 inverse of a rigid matrix is written as the rigid inverse [R^T, -R^T t] (equal to rounding).
// Eigen's JacobiSVD is replaced by a one-sided Jacobi SVD of its own (below); only the metrics, not the transform, are
// defined where the cross-covariance is rank deficient.
#pragma once
#include <cmath>
#include <cstdint>
#include <stdexcept>
#include <vector>

#include "../../oracle/orc_math.h"

namespace orc {
namespace eval {

struct Rt {   // a rigid 4×4 matrix [R t; 0 1]
    Mat3 R;
    Vec3 t;
};
inline Rt MatrixOf(const Pose &p) { return {p.pose.quat.normalized().toRotationMatrix(), p.pose.tr}; }   // TPose::Matrix
inline Vec3 MulVec(const Mat3 &R, const Vec3 &v) {
    return {R(0, 0) * v.x + R(0, 1) * v.y + R(0, 2) * v.z, R(1, 0) * v.x + R(1, 1) * v.y + R(1, 2) * v.z,
            R(2, 0) * v.x + R(2, 1) * v.y + R(2, 2) * v.z};
}
inline Rt Inverse(const Rt &a) {
    const Mat3 Rt_ = a.R.transpose();
    return {Rt_, -MulVec(Rt_, a.t)};
}
inline Rt Mul(const Rt &a, const Rt &b) { return {a.R * b.R, MulVec(a.R, b.t) + a.t}; }

struct KittiErrors {
    std::vector<std::pair<double, double>> tab_errors;
    double mean_rpe = 0, mean_ape = 0, max_ape = 0, mean_local_err = 0, max_local_err = 0;
    int64_t index_max_local_err = 0;
};

// trajectory_distances (eval.cxx:19-24): |(poses[i-1] - poses[i]).t|
inline std::vector<double> KittiDistances(const std::vector<Pose> &gt) {
    std::vector<double> dist(1, 0.0);
    for (size_t i = 1; i < gt.size(); ++i) dist.push_back(dist[i - 1] + (gt[i - 1].pose.tr - gt[i].pose.tr).norm());
    return dist;
}

inline KittiErrors EvaluatePoses(const std::vector<Pose> &gt, const std::vector<Pose> &est,
                                 const std::vector<double> &lengths) {
    if (gt.empty() || est.size() != gt.size()) throw std::invalid_argument("Couldn't evaluate (all) poses");
    if (lengths.empty()) throw std::invalid_argument("empty length list");
    const size_t n = gt.size();
    KittiErrors e;
    for (size_t i = 0; i < n; ++i) {   // APE
        const double ape = Mul(Inverse(MatrixOf(est[i])), MatrixOf(gt[i])).t.norm();
        e.mean_ape += ape;
        if (e.max_ape < ape) e.max_ape = ape;
    }
    e.mean_ape /= (double) n;
    for (size_t i = 1; i < n; ++i) {   // local error
        const double loc = std::fabs((gt[i].pose.tr - gt[i - 1].pose.tr).norm() - (est[i].pose.tr - est[i - 1].pose.tr).norm());
        e.mean_local_err += loc;
        if (e.max_local_err < loc) {
            e.max_local_err = loc;
            e.index_max_local_err = (int64_t) i;
        }
    }
    e.mean_local_err /= (double) (n - 1);
    // ComputeMeanRPE, step size 10
    const std::vector<double> dist = KittiDistances(gt);
    int num_total = 0;
    double mean_rpe = 0;
    for (size_t first = 0; first < n; first += 10) {
        for (double len : lengths) {
            long last = -1;
            for (size_t i = first; i < n; ++i)
                if (dist[i] > dist[first] + len) {
                    last = (long) i;
                    break;
                }
            if (last == -1) continue;
            const Rt dg = Mul(Inverse(MatrixOf(gt[first])), MatrixOf(gt[last]));
            const Rt de = Mul(Inverse(MatrixOf(est[first])), MatrixOf(est[last]));
            const Rt E = Mul(Inverse(de), dg);
            const double t_err = E.t.norm();
            const double d = 0.5 * (E.R(0, 0) + E.R(1, 1) + E.R(2, 2) - 1.0);
            const double r_err = std::acos(std::max(std::min(d, 1.0), -1.0));
            e.tab_errors.emplace_back(t_err / len, r_err / len);
            mean_rpe += t_err / len;
            num_total++;
        }
    }
    e.mean_rpe = (mean_rpe / (double) num_total) * 100.0;
    return e;
}

// ---- OrthogonalProcrustes -------------------------------------------------------------------------------------------
// A = U diag(s) V^T, s decreasing, by one-sided Jacobi: rotate pairs of columns of A (and V) until every pair is
// orthogonal. A column of norm <= 1e-13 of the largest is completed to a right-handed orthonormal U; A = 0 → U = V = I.
inline void SVD3(const Mat3 &Ain, Mat3 &U, Mat3 &V) {
    Mat3 A = Ain;
    V = Mat3();
    for (int i = 0; i < 3; ++i) V(i, i) = 1.0;
    const int P[3] = {0, 0, 1}, Q[3] = {1, 2, 2};
    for (int sweep = 0; sweep < 16; ++sweep) {
        bool rotated = false;
        for (int k = 0; k < 3; ++k) {
            const int p = P[k], q = Q[k];
            double al = 0, be = 0, ga = 0;
            for (int r = 0; r < 3; ++r) {
                al += A(r, p) * A(r, p);
                be += A(r, q) * A(r, q);
                ga += A(r, p) * A(r, q);
            }
            if (!(std::fabs(ga) > 1e-15 * std::sqrt(al) * std::sqrt(be))) continue;
            rotated = true;
            const double zeta = (be - al) / (2.0 * ga);
            const double t = std::fabs(zeta) > 1e150 ? 0.5 / zeta
                                                     : (zeta >= 0 ? 1.0 : -1.0) / (std::fabs(zeta) + std::sqrt(1.0 + zeta * zeta));
            const double c = 1.0 / std::sqrt(1.0 + t * t), s = c * t;
            for (int r = 0; r < 3; ++r) {
                const double ap = A(r, p), aq = A(r, q);
                A(r, p) = c * ap - s * aq;
                A(r, q) = s * ap + c * aq;
                const double vp = V(r, p), vq = V(r, q);
                V(r, p) = c * vp - s * vq;
                V(r, q) = s * vp + c * vq;
            }
        }
        if (!rotated) break;
    }
    double sv[3];
    for (int j = 0; j < 3; ++j) sv[j] = Vec3(A(0, j), A(1, j), A(2, j)).norm();
    auto swap_cols = [&](int i, int j) {
        std::swap(sv[i], sv[j]);
        for (int r = 0; r < 3; ++r) {
            std::swap(A(r, i), A(r, j));
            std::swap(V(r, i), V(r, j));
        }
    };
    if (sv[1] > sv[0]) swap_cols(0, 1);
    if (sv[2] > sv[1]) swap_cols(1, 2);
    if (sv[1] > sv[0]) swap_cols(0, 1);
    U = Mat3();
    if (!(sv[0] > 0.0)) {
        for (int i = 0; i < 3; ++i) U(i, i) = 1.0;
        return;
    }
    const double tol = 1e-13 * sv[0];
    Vec3 u[3];
    u[0] = Vec3(A(0, 0), A(1, 0), A(2, 0)) * (1.0 / sv[0]);
    if (sv[1] > tol) {
        u[1] = Vec3(A(0, 1), A(1, 1), A(2, 1)) * (1.0 / sv[1]);
    } else {
        const double ax = std::fabs(u[0].x), ay = std::fabs(u[0].y), az = std::fabs(u[0].z);
        const Vec3 e = (ax <= ay && ax <= az) ? Vec3(1, 0, 0) : (ay <= az ? Vec3(0, 1, 0) : Vec3(0, 0, 1));
        const Vec3 w = u[0].cross(e);
        u[1] = w * (1.0 / w.norm());
    }
    u[2] = sv[2] > tol ? Vec3(A(0, 2), A(1, 2), A(2, 2)) * (1.0 / sv[2]) : u[0].cross(u[1]);
    for (int j = 0; j < 3; ++j)
        for (int r = 0; r < 3; ++r) U(r, j) = u[j][r];
}

inline double Det(const Mat3 &R) {
    return R(0, 0) * (R(1, 1) * R(2, 2) - R(1, 2) * R(2, 1)) - R(0, 1) * (R(1, 0) * R(2, 2) - R(1, 2) * R(2, 0)) +
           R(0, 2) * (R(1, 0) * R(2, 1) - R(1, 1) * R(2, 0));
}

inline SE3 OrthogonalProcrustes(const std::vector<Vec3> &ref, const std::vector<Vec3> &tgt) {
    Vec3 cr, ct;
    for (size_t i = 0; i < tgt.size(); ++i) {
        cr += ref[i];
        ct += tgt[i];
    }
    cr = Vec3(cr.x / (double) ref.size(), cr.y / (double) ref.size(), cr.z / (double) ref.size());
    ct = Vec3(ct.x / (double) tgt.size(), ct.y / (double) tgt.size(), ct.z / (double) tgt.size());
    Mat3 M;
    for (size_t i = 0; i < tgt.size(); ++i) {
        const Vec3 dt = tgt[i] - ct, dr = ref[i] - cr;
        for (int p = 0; p < 3; ++p)
            for (int q = 0; q < 3; ++q) M(p, q) += dt[p] * dr[q];
    }
    Mat3 U, V;
    SVD3(M, U, V);
    Mat3 R = U * V.transpose();
    if (Det(R) < 0.) {
        Mat3 D;
        D(0, 0) = D(1, 1) = 1.0;
        D(2, 2) = -1.0;
        R = U * D * V.transpose();
    }
    SE3 T;
    T.quat = Quat::fromRotationMatrix(R).normalized();
    T.tr = ct - T.quat * cr;
    return T;
}

struct Segment {
    double segment_length = 0;
    int64_t start_idx = 0, end_idx = 0;
    double loc_error = 0;
    SE3 rigid_transform;
};

struct Metrics {
    std::vector<Segment> segments;   // the counted ones
    std::vector<double> distances;
    double total_distance = 0, mean_ate = 0, max_ate = 0, segment_mean_ate = 0, segment_mean_ate_ratio = 0;
    int64_t max_ate_idx = -1;
    SE3 rigid_transform;
};

// the distances of ComputeTrajectoryMetrics: |(gt_i.pose.Inverse() * gt_{i+1}.pose).tr|, summed in order
inline std::vector<double> MetricsDistances(const std::vector<Pose> &gt) {
    std::vector<double> dist(1, 0.0);
    double distance = 0.;
    for (size_t i = 0; i + 1 < gt.size(); ++i) {
        distance += (gt[i].pose.Inverse() * gt[i + 1].pose).tr.norm();
        dist.push_back(distance);
    }
    return dist;
}

inline Metrics ComputeTrajectoryMetrics(const std::vector<Pose> &gt, const std::vector<Pose> &est,
                                        double segment_length) {
    if (!(segment_length > 0.)) throw std::invalid_argument("segment_length must be > 0");
    if (gt.size() <= 5) throw std::invalid_argument("Cannot estimate the trajectory metrics with less than 5 poses");
    if (est.size() != gt.size()) throw std::invalid_argument("size mismatch");
    const size_t n = gt.size();
    Metrics m;
    m.distances = MetricsDistances(gt);
    m.total_distance = m.distances.back();
    std::vector<Vec3> ref(n), tgt(n);
    for (size_t i = 0; i < n; ++i) {
        ref[i] = gt[i].pose.tr;
        tgt[i] = est[i].pose.tr;
    }
    m.rigid_transform = OrthogonalProcrustes(ref, tgt);
    for (size_t i = 0; i < n; ++i) {
        const double ate = (m.rigid_transform * ref[i] - tgt[i]).norm();   // quat.normalized() * p + tr
        m.mean_ate += ate;
        if (ate > m.max_ate) {
            m.max_ate_idx = (int64_t) i;
            m.max_ate = ate;
        }
    }
    m.mean_ate /= (double) n;
    Segment cur;
    double last_distance = 0.;
    for (size_t idx = 0; idx < n; ++idx) {
        cur.segment_length = m.distances[idx] - last_distance;
        if (cur.segment_length > segment_length) {
            cur.end_idx = (int64_t) idx;
            const size_t count = 1 + cur.end_idx - cur.start_idx;
            if (count > 5) {
                std::vector<Vec3> r, t;
                for (size_t i = 0; i < count; ++i) {
                    r.push_back(gt[cur.start_idx + i].pose.tr);
                    t.push_back(est[cur.start_idx + i].pose.tr);
                }
                cur.rigid_transform = OrthogonalProcrustes(r, t);
                double max_loc = -1.0;
                for (size_t i = 0; i < count; ++i) {
                    const SE3 p = cur.rigid_transform * gt[cur.start_idx + i].pose;
                    max_loc = std::max((p.tr - est[cur.start_idx + i].pose.tr).norm(), max_loc);
                }
                cur.loc_error = max_loc;
                m.segment_mean_ate_ratio += max_loc / cur.segment_length;
                m.segment_mean_ate += max_loc;
                m.segments.push_back(cur);
            }
            cur.segment_length = 0.;
            cur.start_idx = (int64_t) idx;
            last_distance = m.distances[idx];
        }
    }
    m.segment_mean_ate_ratio /= (double) m.segments.size();
    m.segment_mean_ate /= (double) m.segments.size();
    return m;
}

}  // namespace eval
}  // namespace orc
