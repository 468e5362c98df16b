// ORACLE — TEST INFRASTRUCTURE ONLY. The cticp_synthetic_* entry points of include/cticp.h (and, from
// tests/oracle_trajectory, cticp_trajectory_*), prefixed orc_, restated one point at a time in plain host fp64 from the
// reference's src/SlamCore/experimental/synthetic.cxx: Triangle / Line / Ball / Sphere ComputeDistance and RandomPoint,
// Scene::GeneratePoints(CloseToLocation) and GenerateSensorPoints, SyntheticSensorAcquisition::GenerateFrame and
// GeneratePoses, ApplyUniformNoise. Eigen's ColPivHouseholderQR<Matrix3d> (3.3.4+ / 3.4: column-norm downdates, the
// nonzero-pivot threshold, makeHouseholder, the rank-deficient solve) is restated in Eigen's own loop structure, and the
// random source is the draw contract of include/cticp.h instead of rand(). Built with -ffp-contract=off by
// tests/oracle_synthetic_lib.py into liborc_synthetic.so, one library with the trajectory oracle.
#include "../oracle_trajectory/orc_trajectory.cpp"

#include <algorithm>
#include <array>
#include <cmath>

namespace {

// ---- the draw contract -------------------------------------------------------------------------------------------------
uint64_t SplitMix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
const uint64_t kFramePoints = (1ull << 32) | 1u, kFrameNoise = (1ull << 32) | 2u;
const double kRandMax = 2147483647.0;

struct Draws {   // the draws of one primitive (or pose) of one frame
    uint64_t key;
    Draws(uint64_t seed, uint64_t frame, uint64_t prim) : key(SplitMix64(SplitMix64(SplitMix64(seed) ^ frame) ^ prim)) {}
    uint32_t U(uint64_t point, uint32_t j) const { return (uint32_t) (SplitMix64(key ^ ((point << 3) | j)) >> 33); }
    double Random(uint64_t point, uint32_t j) const {   // Eigen 3.3 internal::random<double>(-1, 1)
        return -1.0 + (2.0 * (double) U(point, j)) / kRandMax;
    }
};

using orc::Vec3;

Vec3 Normalized(const Vec3 &v) {   // Eigen normalized(): v / sqrt(squaredNorm) unless zero
    const double z = v.squaredNorm();
    if (z > 0.0) {
        const double n = std::sqrt(z);
        return {v.x / n, v.y / n, v.z / n};
    }
    return v;
}

// ---- Eigen::ColPivHouseholderQR<Matrix3d> -------------------------------------------------------------------------------
struct ColPivQR {
    double qr[3][3];
    double hcoeffs[3];
    int transpositions[3];
    int indices[3];
    int nonzero_pivots;

    explicit ColPivQR(const std::array<Vec3, 3> &cols) {
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) qr[r][c] = cols[c][r];
        const int rows = 3, size = 3;
        double norms_updated[3], norms_direct[3];
        for (int k = 0; k < 3; ++k) {
            norms_direct[k] = std::sqrt(qr[0][k] * qr[0][k] + qr[1][k] * qr[1][k] + qr[2][k] * qr[2][k]);
            norms_updated[k] = norms_direct[k];
        }
        double max_norm = norms_updated[0];
        for (int k = 1; k < 3; ++k) max_norm = norms_updated[k] > max_norm ? norms_updated[k] : max_norm;
        const double eps = std::numeric_limits<double>::epsilon();
        const double threshold_helper = (max_norm * eps) * (max_norm * eps) / (double) rows;
        const double norm_downdate_threshold = std::sqrt(eps);
        nonzero_pivots = size;
        for (int k = 0; k < size; ++k) {
            int biggest = k;
            for (int j = k + 1; j < 3; ++j)
                if (norms_updated[j] > norms_updated[biggest]) biggest = j;
            const double biggest_sq = norms_updated[biggest] * norms_updated[biggest];
            if (nonzero_pivots == size && biggest_sq < threshold_helper * (double) (rows - k)) nonzero_pivots = k;
            transpositions[k] = biggest;
            if (k != biggest) {
                for (int r = 0; r < 3; ++r) std::swap(qr[r][k], qr[r][biggest]);
                std::swap(norms_updated[k], norms_updated[biggest]);
                std::swap(norms_direct[k], norms_direct[biggest]);
            }
            // makeHouseholderInPlace on column k, rows k..2
            double tail_sq = 0.0;
            bool first = true;
            for (int r = k + 1; r < 3; ++r) {
                tail_sq = first ? qr[r][k] * qr[r][k] : tail_sq + qr[r][k] * qr[r][k];
                first = false;
            }
            const double c0 = qr[k][k];
            double beta, tau;
            if (tail_sq <= std::numeric_limits<double>::min()) {
                tau = 0.0;
                beta = c0;
                for (int r = k + 1; r < 3; ++r) qr[r][k] = 0.0;
            } else {
                beta = std::sqrt(c0 * c0 + tail_sq);
                if (c0 >= 0.0) beta = -beta;
                for (int r = k + 1; r < 3; ++r) qr[r][k] = qr[r][k] / (c0 - beta);
                tau = (beta - c0) / beta;
            }
            hcoeffs[k] = tau;
            qr[k][k] = beta;
            // bottomRightCorner(rows - k, cols - k - 1).applyHouseholderOnTheLeft(essential, tau)
            if (k + 1 < 3 && rows - k > 1 && tau != 0.0) {
                for (int j = k + 1; j < 3; ++j) {
                    double tmp = 0.0;
                    bool f = true;
                    for (int r = k + 1; r < 3; ++r) {
                        tmp = f ? qr[r][k] * qr[r][j] : tmp + qr[r][k] * qr[r][j];
                        f = false;
                    }
                    tmp += qr[k][j];
                    qr[k][j] -= tau * tmp;
                    for (int r = k + 1; r < 3; ++r) qr[r][j] -= (tau * qr[r][k]) * tmp;
                }
            }
            for (int j = k + 1; j < 3; ++j) {
                if (norms_updated[j] != 0.0) {
                    double temp = std::abs(qr[k][j]) / norms_updated[j];
                    temp = (1.0 + temp) * (1.0 - temp);
                    temp = temp < 0.0 ? 0.0 : temp;
                    const double ratio = norms_updated[j] / norms_direct[j];
                    const double temp2 = temp * (ratio * ratio);
                    if (temp2 <= norm_downdate_threshold) {
                        double s = 0.0;
                        bool f = true;
                        for (int r = k + 1; r < 3; ++r) {
                            s = f ? qr[r][j] * qr[r][j] : s + qr[r][j] * qr[r][j];
                            f = false;
                        }
                        norms_direct[j] = std::sqrt(s);
                        norms_updated[j] = norms_direct[j];
                    } else {
                        norms_updated[j] *= std::sqrt(temp);
                    }
                }
            }
        }
        for (int i = 0; i < 3; ++i) indices[i] = i;
        for (int k = 0; k < size; ++k) std::swap(indices[k], indices[transpositions[k]]);
    }

    Vec3 Solve(const Vec3 &b) const {
        double c[3] = {b.x, b.y, b.z};
        Vec3 dst;
        if (nonzero_pivots == 0) return Vec3(0, 0, 0);
        for (int k = 0; k < nonzero_pivots; ++k) {   // householderQ().setLength(np).adjoint(): H_0 first
            const int len = 3 - k;
            if (len == 1) {
                c[k] *= 1.0 - hcoeffs[k];
            } else if (hcoeffs[k] != 0.0) {
                double tmp = 0.0;
                bool f = true;
                for (int r = k + 1; r < 3; ++r) {
                    tmp = f ? qr[r][k] * c[r] : tmp + qr[r][k] * c[r];
                    f = false;
                }
                tmp += c[k];
                c[k] -= hcoeffs[k] * tmp;
                for (int r = k + 1; r < 3; ++r) c[r] -= (hcoeffs[k] * qr[r][k]) * tmp;
            }
        }
        // triangular_solve_vector<Upper, ColMajor>: the panel loop, from the last row up
        for (int k = 0; k < nonzero_pivots; ++k) {
            const int i = nonzero_pivots - k - 1;
            if (c[i] != 0.0) {
                c[i] /= qr[i][i];
                for (int s = 0; s < i; ++s) c[s] -= c[i] * qr[s][i];
            }
        }
        for (int i = 0; i < nonzero_pivots; ++i) dst[indices[i]] = c[i];
        for (int i = nonzero_pivots; i < 3; ++i) dst[indices[i]] = 0.0;
        return dst;
    }
};

// ---- primitives -----------------------------------------------------------------------------------------------------
struct Primitive {
    int kind;
    std::array<Vec3, 3> points;
    Vec3 center;
    double radius = 0.0;
    ColPivQR *qr = nullptr;

    Vec3 Normal() const { return Normalized((points[0] - points[2]).cross(points[1] - points[2])); }
    Vec3 Direction() const { return Normalized(points[0] - points[1]); }

    double Distance(const Vec3 &point) const {
        switch (kind) {
            case CTICP_SYN_TRIANGLE: {
                auto min_distance = [&](const Vec3 &q) {
                    double d = std::numeric_limits<double>::max();
                    for (int i = 0; i < 3; ++i) d = std::min((points[i] - q).norm(), d);
                    const Vec3 s = (points[0] + points[1]) + points[2];
                    const Vec3 bary(s.x / 3.0, s.y / 3.0, s.z / 3.0);
                    return std::min(d, (bary - q).norm());
                };
                const Vec3 n = Normal();
                const double ptp = (point - points[2]).dot(n);
                const Vec3 projected = point - n * ptp;
                const Vec3 coeffs = qr->Solve(projected);
                bool in_triangle = true;
                for (int i = 0; i < 3; ++i)
                    if (coeffs[i] < 0. || coeffs[i] > 1.) {
                        in_triangle = false;
                        break;
                    }
                return std::min(std::abs(ptp) + (in_triangle ? 0. : min_distance(projected)), min_distance(point));
            }
            case CTICP_SYN_LINE: {
                auto min_distance = [&](const Vec3 &q) {
                    double d = std::numeric_limits<double>::max();
                    for (int i = 0; i < 2; ++i) d = std::min(d, (q - points[i]).norm());
                    const Vec3 s = points[0] + points[1];
                    const Vec3 bary(s.x / 2.0, s.y / 2.0, s.z / 2.0);
                    return std::min(d, (q - bary).norm());
                };
                const Vec3 d = Direction();
                const double s = (point - points[0]).dot(d);
                const Vec3 projected = points[0] + d * std::sqrt(s * s);   // ((x - p0)^T d).norm() of a 1x1 product
                const double distance_to_line = (projected - point).norm();
                const double norm_ab = (points[0] - points[1]).dot(d);
                double norm_a_point = (points[0] - projected).dot(d);
                norm_a_point /= norm_ab;
                const bool outside_segment = norm_a_point > 1.0 || norm_a_point < 0.;
                return std::min(min_distance(point), distance_to_line + (outside_segment ? min_distance(projected) : 0.));
            }
            case CTICP_SYN_BALL:
                return std::max(0., (point - center).norm() - radius);
            default:
                return std::abs((point - center).norm() - radius);
        }
    }

    Vec3 RandomPoint(const Draws &dr, uint64_t i) const {
        switch (kind) {
            case CTICP_SYN_TRIANGLE: {
                double c[3];
                for (uint32_t j = 0; j < 3; ++j) c[j] = std::pow(dr.Random(i, j) + 1.0, 1.5);
                const double sum = (c[0] + c[1]) + c[2];
                for (double &v : c) v /= sum;
                Vec3 p(0, 0, 0);
                for (int j = 0; j < 3; ++j) p += points[j] * c[j];
                return p;
            }
            case CTICP_SYN_LINE: {
                double c0 = std::abs(dr.Random(i, 0)), c1 = std::abs(dr.Random(i, 1));
                const double sum = c0 + c1;
                c0 /= sum;
                c1 /= sum;
                return points[0] * c0 + points[1] * c1;
            }
            case CTICP_SYN_BALL: {
                const Vec3 r(dr.Random(i, 0), dr.Random(i, 1), dr.Random(i, 2));
                const double r3 = dr.Random(i, 3);
                return center + Normalized(r) * radius * std::abs(r3);
            }
            default:
                return center + Normalized(Vec3(dr.Random(i, 0), dr.Random(i, 1), dr.Random(i, 2))) * radius;
        }
    }
};

}  // namespace

struct orc_synthetic_scene {
    std::vector<Primitive> prims;
    std::vector<std::unique_ptr<ColPivQR>> factors;
};

namespace {

// Scene::GenerateSensorPoints of one frame, appended to the outputs (world, raw, t, primitive, point)
struct Out {
    std::vector<Vec3> world, raw;
    std::vector<double> t;
    std::vector<uint32_t> prim, point;
};

void GenerateFrame(const orc_synthetic_scene &s, const orc::LinearContinuousTrajectory &traj,
                   const cticp_synthetic_frame &f, size_t n, double d, uint64_t seed, Out &o) {
    const orc::Pose begin = traj.InterpolatePose(f.begin_ts), end = traj.InterpolatePose(f.end_ts);
    for (size_t p = 0; p < s.prims.size(); ++p) {
        const Primitive &P = s.prims[p];
        if (!(P.Distance(begin.pose.tr) < d || P.Distance(end.pose.tr) < d)) continue;
        const Draws dr(seed, f.frame_id, p);
        for (size_t i = 0; i < n; ++i) {
            const Vec3 world = P.RandomPoint(dr, i);
            const double alpha = (double) dr.U(i, 4) / kRandMax;
            const double t = begin.dest_timestamp * (1 - alpha) + alpha * end.dest_timestamp;
            const Vec3 raw = begin.InterpolatePoseAlpha(end, alpha).pose.Inverse() * world;
            if (raw.norm() < d) {
                o.world.push_back(world);
                o.raw.push_back(raw);
                o.t.push_back(t);
                o.prim.push_back((uint32_t) p);
                o.point.push_back((uint32_t) i);
            }
        }
    }
}

void Store(unsigned char *rec, const cticp_cloud_sink &sink, const Vec3 &v, double t) {
    if (sink.xyz_dtype == CTICP_DTYPE_FLOAT32) {
        const float f[3] = {(float) v.x, (float) v.y, (float) v.z};
        memcpy(rec + sink.xyz_offset, f, 12);
    } else {
        const double f[3] = {v.x, v.y, v.z};
        memcpy(rec + sink.xyz_offset, f, 24);
    }
    if (sink.t_dtype == CTICP_DTYPE_FLOAT32) {
        const float ft = (float) t;
        memcpy(rec + sink.t_offset, &ft, 4);
    } else if (sink.t_dtype == CTICP_DTYPE_FLOAT64) {
        memcpy(rec + sink.t_offset, &t, 8);
    }
}

}  // namespace

extern "C" {

int orc_synthetic_scene_create(const double *triangles, size_t nt, const double *lines, size_t nl, const double *spheres,
                               size_t ns, const double *balls, size_t nb, int device, orc_synthetic_scene **out) {
    (void) device;
    return Guard([&] {
        if (!out) throw std::invalid_argument("null argument");
        auto s = std::make_unique<orc_synthetic_scene>();
        auto finite = [](const double *v, size_t n) {
            for (size_t i = 0; i < n; ++i)
                if (!std::isfinite(v[i])) throw std::invalid_argument("a value is not finite");
        };
        finite(triangles, 9 * nt);
        finite(lines, 6 * nl);
        finite(spheres, 4 * ns);
        finite(balls, 4 * nb);
        for (size_t i = 0; i < nt; ++i) {
            Primitive P{CTICP_SYN_TRIANGLE};
            for (int k = 0; k < 3; ++k) P.points[k] = Vec3(triangles[9 * i + 3 * k], triangles[9 * i + 3 * k + 1],
                                                           triangles[9 * i + 3 * k + 2]);
            s->factors.push_back(std::make_unique<ColPivQR>(P.points));
            P.qr = s->factors.back().get();
            s->prims.push_back(P);
        }
        for (size_t i = 0; i < nl; ++i) {
            Primitive P{CTICP_SYN_LINE};
            for (int k = 0; k < 2; ++k) P.points[k] = Vec3(lines[6 * i + 3 * k], lines[6 * i + 3 * k + 1], lines[6 * i + 3 * k + 2]);
            s->prims.push_back(P);
        }
        for (int kind : {CTICP_SYN_SPHERE, CTICP_SYN_BALL}) {
            const double *v = kind == CTICP_SYN_SPHERE ? spheres : balls;
            const size_t n = kind == CTICP_SYN_SPHERE ? ns : nb;
            for (size_t i = 0; i < n; ++i) {
                if (v[4 * i + 3] < 0.0) throw std::invalid_argument("a radius is negative");
                Primitive P{kind};
                P.center = Vec3(v[4 * i], v[4 * i + 1], v[4 * i + 2]);
                P.radius = v[4 * i + 3];
                s->prims.push_back(P);
            }
        }
        *out = s.release();
        return 0;
    });
}
void orc_synthetic_scene_destroy(orc_synthetic_scene *s) { delete s; }
int64_t orc_synthetic_scene_num_primitives(orc_synthetic_scene *s) { return (int64_t) s->prims.size(); }
int orc_synthetic_scene_distance(orc_synthetic_scene *s, const double *points, size_t m, double *out) {
    return Guard([&] {
        const size_t np = s->prims.size();
        for (size_t q = 0; q < m; ++q)
            for (size_t p = 0; p < np; ++p)
                out[q * np + p] = s->prims[p].Distance(Vec3(points[3 * q], points[3 * q + 1], points[3 * q + 2]));
        return 0;
    });
}
int64_t orc_synthetic_generate_points(orc_synthetic_scene *s, size_t n, const double *location, double distance,
                                      uint64_t seed, double *xyz, size_t cap, uint32_t *src_index) {
    size_t count = 0;
    int rc = Guard([&] {
        for (size_t p = 0; p < s->prims.size(); ++p) {
            const Primitive &P = s->prims[p];
            if (location && !(P.Distance(Vec3(location[0], location[1], location[2])) <= distance)) continue;
            const Draws dr(seed, kFramePoints, p);
            for (size_t i = 0; i < n; ++i, ++count) {
                const Vec3 w = P.RandomPoint(dr, i);
                if (count >= cap) continue;
                if (xyz) {
                    xyz[3 * count] = w.x;
                    xyz[3 * count + 1] = w.y;
                    xyz[3 * count + 2] = w.z;
                }
                if (src_index) {
                    src_index[2 * count] = (uint32_t) p;
                    src_index[2 * count + 1] = (uint32_t) i;
                }
            }
        }
        return 0;
    });
    return rc < 0 ? rc : (int64_t) count;
}
int64_t orc_synthetic_generate_frames(orc_synthetic_scene *s, orc_trajectory *t, const cticp_synthetic_frame *frames,
                                      size_t m, size_t n, double distance, uint64_t seed, const cticp_cloud_sink *sink,
                                      uint32_t *src_index, uint64_t *frame_ends) {
    size_t count = 0;
    int rc = Guard([&] {
        if (!s || !t || !sink || (m && (!frames || !frame_ends))) throw std::invalid_argument("null argument");
        if (!(distance > 0.0) || !std::isfinite(distance)) throw std::invalid_argument("distance");
        if (n < 2) throw std::invalid_argument("Need to generate at least two points");
        for (size_t k = 0; k < m; ++k)
            if (!(frames[k].begin_ts <= frames[k].end_ts)) throw std::invalid_argument("begin_ts > end_ts");
        Out o;
        std::vector<uint64_t> ends(m);
        for (size_t k = 0; k < m; ++k) {
            GenerateFrame(*s, t->t, frames[k], n, distance, seed, o);
            ends[k] = o.t.size();
        }
        count = o.t.size();
        const size_t w = std::min<size_t>(count, sink->capacity_points);
        for (size_t i = 0; i < w; ++i) {
            if (sink->data)
                Store(static_cast<unsigned char *>(sink->data) + i * sink->point_step, *sink,
                      sink->world ? o.world[i] : o.raw[i], o.t[i]);
            if (src_index) {
                src_index[2 * i] = o.prim[i];
                src_index[2 * i + 1] = o.point[i];
            }
        }
        std::copy(ends.begin(), ends.end(), frame_ends);
        return 0;
    });
    return rc < 0 ? rc : (int64_t) count;
}
int64_t orc_synthetic_generate_poses(orc_trajectory *t, double frequency, cticp_pose *out, size_t cap) {
    int64_t count = 0;
    int rc = Guard([&] {
        const double step = 1. / frequency;
        double current = t->t.MinTimestamp();
        const double max_timestamp = t->t.MaxTimestamp();
        if (!(max_timestamp - current > step)) throw std::invalid_argument("The interval between the first and last poses");
        std::vector<cticp_pose> poses;
        while (current <= max_timestamp) {
            poses.push_back(ToC(t->t.InterpolatePose(current)));
            current += step;
        }
        for (size_t i = 0; i < poses.size() && i < cap; ++i) out[i] = poses[i];
        count = (int64_t) poses.size();
        return 0;
    });
    return rc < 0 ? rc : count;
}
int orc_apply_uniform_noise(cticp_pose *poses, size_t n, double scale_rot_deg, double scale_trans_m, uint64_t seed) {
    for (size_t i = 0; i < n; ++i) {
        const Draws dr(seed, kFrameNoise, i);
        const Vec3 rot(dr.Random(0, 0) * scale_rot_deg * M_PI / 180.0, dr.Random(0, 1) * scale_rot_deg * M_PI / 180.0,
                       dr.Random(0, 2) * scale_rot_deg * M_PI / 180.0);
        const Vec3 tr(dr.Random(0, 3) * scale_trans_m, dr.Random(0, 4) * scale_trans_m, dr.Random(0, 5) * scale_trans_m);
        auto angle_axis = [](double angle, int axis) {   // Quaternion(AngleAxis(angle, Unit(axis)))
            const double ha = 0.5 * angle, s = std::sin(ha);
            return orc::Quat(s * (axis == 0 ? 1.0 : 0.0), s * (axis == 1 ? 1.0 : 0.0), s * (axis == 2 ? 1.0 : 0.0),
                             std::cos(ha));
        };
        const orc::Quat q = angle_axis(rot.x, 0) * angle_axis(rot.y, 1) * angle_axis(rot.z, 2);
        const orc::SE3 noise(q.normalized(), tr);
        orc::Pose p = FromC(poses[i]);
        p.pose = noise * p.pose;
        poses[i] = ToC(p);
    }
    return 0;
}

}  // extern "C"
