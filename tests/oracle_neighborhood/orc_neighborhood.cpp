// orc_neighborhood.cpp — a plain C++ restatement of slam::TNeighborhood (include/SlamCore/experimental/neighborhood.h),
// written from its documented behaviour: the k-nearest search of nanoflann's KDTreeSingleIndexAdaptor with the
// reference's KNNRadiusResultSet, by brute force over the points in index order (nanoflann's L2_Simple_Adaptor d2,
// the leaf test dist < worstDist() and addPoint's insertion, so equal d2 keep index order), ComputeNeighborhood's
// description twice (the reference's uncentred fp64 sums, and centred in long double), Eigen's 3x3 cofactor determinant
// and ClassifyNeighborhood. The SVD is oracle/orc_math.h's SymmetricSVD3. Built with -ffp-contract=off. TEST INFRASTRUCTURE.
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../include/cticp.h"
#include "../../oracle/orc_math.h"

namespace {

bool Finite(const double *p) { return std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]); }

// nanoflann::KNNRadiusResultSet (neighborhood.h:12-41, 323-357)
struct ResultSet {
    double max_radius;
    size_t capacity, count = 0;
    uint64_t *indices;
    double *dists;
    double WorstDist() const { return std::min(dists[capacity - 1], max_radius); }
    void AddPoint(double dist, uint64_t index) {
        if (dist > max_radius) return;
        size_t i;
        for (i = count; i > 0; --i) {
            if (dists[i - 1] > dist) {
                if (i < capacity) {
                    dists[i] = dists[i - 1];
                    indices[i] = indices[i - 1];
                }
            } else
                break;
        }
        if (i < capacity) {
            dists[i] = dist;
            indices[i] = index;
        }
        if (count < capacity) count++;
    }
};

double Cofactor3(const double c[6]) {   // Eigen's determinant of a 3x3: m00 (m11 m22 - m12 m21) - m01 (...) + m02 (...)
    const double m00 = c[0], m01 = c[1], m02 = c[2], m10 = c[1], m11 = c[3], m12 = c[4], m20 = c[2], m21 = c[4], m22 = c[5];
    return m00 * (m11 * m22 - m12 * m21) - m01 * (m10 * m22 - m12 * m20) + m02 * (m10 * m21 - m11 * m20);
}

void Describe(const double *pts, size_t n, const double *centre, int values, double lin_t, double plan_t, int centred,
              cticp_neighborhood_description *d) {
    std::memset(d, 0, sizeof(*d));
    d->planarity = d->linearity = d->a2D = d->cov_det = -1.0;
    d->type = CTICP_NB_TYPE_NONE;
    if (n < 5) return;   // ComputeNeighborhood returns early; ClassifyNeighborhood then sees NO_VALUES
    double bary[3], cov[6];
    if (!centred) {   // neighborhood.h:231-244
        double b[3] = {0, 0, 0}, c[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
        for (size_t i = 0; i < n; ++i) {
            const double *p = pts + 3 * i;
            for (int a = 0; a < 3; ++a) {
                b[a] += p[a];
                for (int e = 0; e < 3; ++e) c[a][e] += p[a] * p[e];
            }
        }
        for (int a = 0; a < 3; ++a) b[a] /= (double) n;
        for (int a = 0; a < 3; ++a)
            for (int e = 0; e < 3; ++e) c[a][e] = c[a][e] / (double) n - b[a] * b[e];
        for (int a = 0; a < 3; ++a) bary[a] = b[a];
        const int ij[6][2] = {{0, 0}, {0, 1}, {0, 2}, {1, 1}, {1, 2}, {2, 2}};
        for (int t = 0; t < 6; ++t) cov[t] = c[ij[t][0]][ij[t][1]];
    } else {
        const double *o = centre ? centre : pts;
        long double s[3] = {0, 0, 0}, ss[6] = {0, 0, 0, 0, 0, 0};
        for (size_t i = 0; i < n; ++i) {
            long double r[3];
            for (int a = 0; a < 3; ++a) r[a] = (long double) pts[3 * i + a] - (long double) o[a];
            for (int a = 0; a < 3; ++a) s[a] += r[a];
            ss[0] += r[0] * r[0]; ss[1] += r[0] * r[1]; ss[2] += r[0] * r[2];
            ss[3] += r[1] * r[1]; ss[4] += r[1] * r[2]; ss[5] += r[2] * r[2];
        }
        long double m[3];
        for (int a = 0; a < 3; ++a) m[a] = s[a] / (long double) n;
        const int ij[6][2] = {{0, 0}, {0, 1}, {0, 2}, {1, 1}, {1, 2}, {2, 2}};
        for (int t = 0; t < 6; ++t) cov[t] = (double) (ss[t] / (long double) n - m[ij[t][0]] * m[ij[t][1]]);
        for (int a = 0; a < 3; ++a) bary[a] = (double) ((long double) o[a] + m[a]);
    }
    orc::Mat3 C, V;
    const int ij[6][2] = {{0, 0}, {0, 1}, {0, 2}, {1, 1}, {1, 2}, {2, 2}};
    for (int t = 0; t < 6; ++t) C(ij[t][0], ij[t][1]) = C(ij[t][1], ij[t][0]) = cov[t];
    double sv[3];
    orc::SymmetricSVD3(C, sv, V);   // singular values already abs, descending
    for (int a = 0; a < 3; ++a) d->barycenter[a] = bary[a];
    for (int t = 0; t < 6; ++t) d->covariance[t] = cov[t];
    if (values & CTICP_NB_LINE)
        for (int a = 0; a < 3; ++a) d->line[a] = V(a, 0);
    if (values & CTICP_NB_NORMAL)
        for (int a = 0; a < 3; ++a) d->normal[a] = V(a, 2);
    if (values & CTICP_NB_LINEARITY) d->linearity = (sv[0] - sv[1]) / sv[0];
    if (values & CTICP_NB_PLANARITY) d->planarity = (sv[1] - sv[2]) / sv[0];
    if (values & CTICP_NB_A2D) d->a2D = (std::sqrt(sv[1]) - std::sqrt(sv[2])) / std::sqrt(sv[0]);
    if (values & CTICP_NB_COV_DET) d->cov_det = Cofactor3(cov);
    d->is_valid = 1;
    // ClassifyNeighborhood(linearity_thresh, planarity_thresh), neighborhood.h:269-282
    if ((values & CTICP_NB_PLANARITY) && (values & CTICP_NB_LINEARITY)) {
        if (d->planarity > plan_t) d->type = CTICP_NB_TYPE_PLANAR;
        else if (d->linearity > lin_t) d->type = CTICP_NB_TYPE_LINEAR;
    } else if ((values & CTICP_NB_COV_DET) && n > 5) {
        d->type = CTICP_NB_TYPE_VOLUMIC;
    }
}

}  // namespace

extern "C" {

// k nearest of m queries (NULL: the points themselves) among n points: indices / d2 (m k; ~0 / +inf past the count)
void orn_search(const double *pts, size_t n, const double *queries, size_t m, int k, double max_radius, uint64_t *indices,
                double *d2, int32_t *counts) {
    for (size_t q = 0; q < m; ++q) {
        const double *qp = queries ? queries + 3 * q : pts + 3 * q;
        ResultSet rs{max_radius, (size_t) k, 0, indices + q * k, d2 + q * k};
        for (int j = 0; j < k; ++j) {
            rs.indices[j] = ~0ull;
            rs.dists[j] = INFINITY;
        }
        rs.dists[k - 1] = DBL_MAX;   // KNNRadiusResultSet::init
        if (Finite(qp))
            for (size_t i = 0; i < n; ++i) {
                const double *p = pts + 3 * i;
                if (!Finite(p)) continue;
                double dist = 0.0;   // L2_Simple_Adaptor::evalMetric: result += diff * diff, diff = query - point
                for (int a = 0; a < 3; ++a) {
                    const double diff = qp[a] - p[a];
                    dist += diff * diff;
                }
                if (dist < rs.WorstDist()) rs.AddPoint(dist, i);
            }
        counts[q] = (int32_t) rs.count;
        for (size_t j = rs.count; j < (size_t) k; ++j) {
            rs.indices[j] = ~0ull;
            rs.dists[j] = INFINITY;
        }
    }
}

// ComputeNeighborhood(values) + ClassifyNeighborhood of n points; centred 0: the reference's uncentred fp64 sums,
// 1: centred on `centre` (NULL: the first point) in long double
void orn_describe(const double *pts, size_t n, const double *centre, int values, double lin_t, double plan_t,
                  int centred, cticp_neighborhood_description *out) {
    Describe(pts, n, centre, values, lin_t, plan_t, centred, out);
}

}  // extern "C"
