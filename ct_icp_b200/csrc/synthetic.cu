// synthetic.cu — slam::Scene and slam::SyntheticSensorAcquisition on the device.
//
// Reference: src/SlamCore/experimental/synthetic.cxx (ComputeDistance :62-91, :116-139, :150-180; RandomPoint :94-103,
// :142-146, :156-186; GeneratePointsCloseToLocation / GeneratePoints :249-285; GenerateSensorPoints :293-327;
// GenerateFrame :365-380), include/SlamCore/experimental/synthetic.h (Normal, Barycenter, Direction).
//
// This file is compiled with -fmad=false: every Distance is the fp64 arithmetic a host loop does, operation for
// operation, so the selection decisions equal a host restatement's bit for bit. A call runs three steps on the scene's
// stream:
//   1. select: one thread per (frame, primitive) evaluates the two Distances;
//   2. generate + compact: one pass over tiles of (frame, primitive, 512 points) in that order, tiles taken from an atomic
//      ticket. Each lane makes its draws and computes its world point, the pose at alpha and the raw point; a tile's
//      kept points are numbered by a block scan and placed by the decoupled look-back of tile_lookback.cuh, so the output
//      is in (frame, primitive, point) order whatever the schedule;
//   3. the last tile of a frame writes its end.
#include "synthetic.h"

#include <algorithm>
#include <cmath>
#include <limits>
#include <stdexcept>
#include <string>

#include "device_checks.h"
#include "device_map.h"
#include "record_io.cuh"
#include "scan_pack.cuh"
#include "se3.cuh"
#include "tile_lookback.cuh"
#include "trajectory.h"

namespace cticp {

namespace {

constexpr int kThreads = 256;
constexpr int kPerThread = 2;
constexpr uint64_t kTile = kThreads * kPerThread;   // points of one tile
constexpr double kRandMax = 2147483647.0;
constexpr uint64_t kKeyPoints = (1ull << 32) | 1u;  // the frame slot of the calls without a frame (frame ids are 32-bit)
constexpr uint64_t kKeyNoise = (1ull << 32) | 2u;

// ---- the draw order contract (DESIGN.md §4) ---------------------------------------------------------------------------
CT_HD uint64_t prim_key(uint64_t seed, uint64_t frame_key, uint64_t prim) {
    return splitmix64(splitmix64(splitmix64(seed) ^ frame_key) ^ prim);
}
CT_HD uint32_t draw(uint64_t pkey, uint64_t point, uint32_t j) {
    return (uint32_t) (splitmix64(pkey ^ ((point << 3) | j)) >> 33);
}
CT_HD double rnd(uint32_t u) { return -1.0 + (2.0 * (double) u) / kRandMax; }   // Eigen 3.3 random<double>(-1, 1)

// ---- Distance ----------------------------------------------------------------------------------------------------------
CT_HD double norm3(double x, double y, double z) { return sqrt(x * x + y * y + z * z); }
CT_HD double dmin(double a, double b) { return b < a ? b : a; }   // std::min(a, b)
CT_HD double dmax(double a, double b) { return a < b ? b : a; }   // std::max(a, b)

// the triangle's compute_min_distance: corners in order, then the barycentre
CT_HD double tri_corner_distance(const SynPrim &P, double x, double y, double z) {
    double d = std::numeric_limits<double>::max();
    for (int i = 0; i < 3; ++i) d = dmin(norm3(P.p[i][0] - x, P.p[i][1] - y, P.p[i][2] - z), d);
    return dmin(d, norm3(P.b[0] - x, P.b[1] - y, P.b[2] - z));
}
CT_HD double line_corner_distance(const SynPrim &P, double x, double y, double z) {
    double d = std::numeric_limits<double>::max();
    for (int i = 0; i < 2; ++i) d = dmin(d, norm3(x - P.p[i][0], y - P.p[i][1], z - P.p[i][2]));
    return dmin(d, norm3(x - P.b[0], y - P.b[1], z - P.b[2]));
}

// A.colPivHouseholderQr().solve(b) with the factor of the scene: Q^T b (H_0 first), back-substitution on the leading
// rank × rank block of R as Eigen's triangular solver runs it (column by column, skipping a zero), the free coefficients 0,
// written back through the column permutation
CT_HD void qr_solve(const SynPrim &P, const double b[3], double out[3]) {
    double c[3] = {b[0], b[1], b[2]};
    const int np = P.rank;
    for (int k = 0; k < np; ++k) {
        if (k == 2) {
            c[2] *= 1.0 - P.tau[2];
        } else if (P.tau[k] != 0.0) {
            double tmp = P.qr[k + 1][k] * c[k + 1];
            if (k == 0) tmp = tmp + P.qr[2][0] * c[2];
            tmp += c[k];
            c[k] -= P.tau[k] * tmp;
            for (int i = k + 1; i < 3; ++i) c[i] -= (P.tau[k] * P.qr[i][k]) * tmp;
        }
    }
    for (int i = np - 1; i >= 0; --i) {
        if (c[i] != 0.0) {
            c[i] /= P.qr[i][i];
            for (int s = 0; s < i; ++s) c[s] -= c[i] * P.qr[s][i];
        }
    }
    for (int i = 0; i < 3; ++i) out[P.perm[i]] = i < np ? c[i] : 0.0;
}

CT_HD double prim_distance(const SynPrim &P, double x, double y, double z) {
    switch (P.kind) {
        case CTICP_SYN_TRIANGLE: {
            const double ptp = (x - P.p[2][0]) * P.n[0] + (y - P.p[2][1]) * P.n[1] + (z - P.p[2][2]) * P.n[2];
            const double pr[3] = {x - ptp * P.n[0], y - ptp * P.n[1], z - ptp * P.n[2]};
            double co[3];
            qr_solve(P, pr, co);
            bool inside = true;
            for (int i = 0; i < 3; ++i)
                if (co[i] < 0.0 || co[i] > 1.0) {
                    inside = false;
                    break;
                }
            return dmin(fabs(ptp) + (inside ? 0.0 : tri_corner_distance(P, pr[0], pr[1], pr[2])),
                        tri_corner_distance(P, x, y, z));
        }
        case CTICP_SYN_LINE: {
            const double *d = P.n;
            const double s = (x - P.p[0][0]) * d[0] + (y - P.p[0][1]) * d[1] + (z - P.p[0][2]) * d[2];
            const double a = sqrt(s * s);   // the norm of a 1 x 1 product
            const double pr[3] = {P.p[0][0] + a * d[0], P.p[0][1] + a * d[1], P.p[0][2] + a * d[2]};
            const double to_line = norm3(pr[0] - x, pr[1] - y, pr[2] - z);
            const double ab = (P.p[0][0] - P.p[1][0]) * d[0] + (P.p[0][1] - P.p[1][1]) * d[1] + (P.p[0][2] - P.p[1][2]) * d[2];
            double ap = (P.p[0][0] - pr[0]) * d[0] + (P.p[0][1] - pr[1]) * d[1] + (P.p[0][2] - pr[2]) * d[2];
            ap /= ab;
            const bool outside = ap > 1.0 || ap < 0.0;
            return dmin(line_corner_distance(P, x, y, z),
                        to_line + (outside ? line_corner_distance(P, pr[0], pr[1], pr[2]) : 0.0));
        }
        case CTICP_SYN_BALL:
            return dmax(0.0, norm3(x - P.p[0][0], y - P.p[0][1], z - P.p[0][2]) - P.radius);
        default:
            return fabs(norm3(x - P.p[0][0], y - P.p[0][1], z - P.p[0][2]) - P.radius);
    }
}

// RandomPoint with the draws of (pkey, point): draws 0..3 as the primitive needs them
__device__ __forceinline__ V3 random_point(const SynPrim &P, uint64_t pkey, uint64_t i) {
    switch (P.kind) {
        case CTICP_SYN_TRIANGLE: {
            double c[3];
            for (int j = 0; j < 3; ++j) c[j] = pow(rnd(draw(pkey, i, j)) + 1.0, 1.5);
            const double s = c[0] + c[1] + c[2];
            for (int j = 0; j < 3; ++j) c[j] /= s;
            V3 r{0.0, 0.0, 0.0};
            for (int j = 0; j < 3; ++j) r = V3{r.x + P.p[j][0] * c[j], r.y + P.p[j][1] * c[j], r.z + P.p[j][2] * c[j]};
            return r;
        }
        case CTICP_SYN_LINE: {
            double c0 = fabs(rnd(draw(pkey, i, 0))), c1 = fabs(rnd(draw(pkey, i, 1)));
            const double s = c0 + c1;
            c0 /= s;
            c1 /= s;
            return V3{P.p[0][0] * c0 + P.p[1][0] * c1, P.p[0][1] * c0 + P.p[1][1] * c1, P.p[0][2] * c0 + P.p[1][2] * c1};
        }
        default: {   // sphere: c + normalized(r) R; ball: c + normalized(r) R |r_3|
            double v[3] = {rnd(draw(pkey, i, 0)), rnd(draw(pkey, i, 1)), rnd(draw(pkey, i, 2))};
            const double z = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
            if (z > 0.0) {
                const double s = sqrt(z);
                for (int j = 0; j < 3; ++j) v[j] /= s;
            }
            if (P.kind == CTICP_SYN_BALL) {
                const double a = fabs(rnd(draw(pkey, i, 3)));
                return V3{P.p[0][0] + v[0] * P.radius * a, P.p[0][1] + v[1] * P.radius * a, P.p[0][2] + v[2] * P.radius * a};
            }
            return V3{P.p[0][0] + v[0] * P.radius, P.p[0][1] + v[1] * P.radius, P.p[0][2] + v[2] * P.radius};
        }
    }
}

__global__ void __launch_bounds__(kThreads) k_distance(const SynPrim *__restrict__ prims, uint32_t np,
                                                       const double *__restrict__ q, uint64_t m, double *__restrict__ out) {
    for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < m * np; i += (uint64_t) gridDim.x * blockDim.x) {
        const uint64_t k = i / np;
        out[i] = prim_distance(prims[i - k * np], q[3 * k], q[3 * k + 1], q[3 * k + 2]);
    }
}

// mode 0: used when Distance(begin.tr) < d || Distance(end.tr) < d (poses: [2 m]); 1: every primitive; 2: Distance(loc) <= d
__global__ void __launch_bounds__(kThreads) k_select(const SynPrim *__restrict__ prims, uint32_t np, uint64_t m, int mode,
                                                     const cticp_pose *__restrict__ poses, double3 loc, double d,
                                                     unsigned char *__restrict__ sel) {
    for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < m * np; i += (uint64_t) gridDim.x * blockDim.x) {
        const uint64_t f = i / np;
        const SynPrim &P = prims[i - f * np];
        bool s = true;
        if (mode == 0) {
            const cticp_pose &b = poses[2 * f], &e = poses[2 * f + 1];
            s = prim_distance(P, b.tr[0], b.tr[1], b.tr[2]) < d || prim_distance(P, e.tr[0], e.tr[1], e.tr[2]) < d;
        } else if (mode == 2) {
            s = prim_distance(P, loc.x, loc.y, loc.z) <= d;
        }
        sel[i] = s ? 1 : 0;
    }
}

struct GenArgs {
    const SynPrim *prims;
    uint32_t np;
    uint64_t n, chunks, tiles;
    const unsigned char *sel;
    const cticp_pose *poses;                 // frames: [2 m] begin, end
    const cticp_synthetic_frame *frames;     // frames: the frame ids; nullptr: the calls without a frame
    uint64_t seed;
    double d;
    unsigned long long *desc;                // [tiles] descriptors, [tiles] the ticket
    uint32_t *src;
    uint64_t *ends;
};

// One tile = (frame f, primitive p, points [c kTile, (c + 1) kTile)); thread j holds points c kTile + kPerThread j + k.
__global__ void __launch_bounds__(kThreads, 2) k_generate(GenArgs g, GenSink sink) {
    __shared__ unsigned long long s_tile;
    __shared__ uint32_t s_warp[kThreads / 32];
    __shared__ uint32_t s_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (;;) {
        if (threadIdx.x == 0) s_tile = atomicAdd(&g.desc[g.tiles], 1ull);
        __syncthreads();
        const unsigned long long tile = s_tile;
        if (tile >= g.tiles) break;
        const uint64_t c = tile % g.chunks, fp = tile / g.chunks;
        const uint64_t f = fp / g.np;
        const uint32_t p = (uint32_t) (fp - f * g.np);
        V3 pts[kPerThread];
        double ts[kPerThread];
        uint32_t keep = 0;   // bit k: point k of this thread is emitted
        if (g.sel[fp]) {
            const SynPrim &P = g.prims[p];
            const uint64_t pkey = prim_key(g.seed, g.frames ? (uint64_t) g.frames[f].frame_id : kKeyPoints, p);
            Q4 qb{}, qe{};
            V3 tb{}, te{};
            double tsb = 0.0, tse = 0.0;
            SlerpConsts sc{};
            if (g.frames) {
                const cticp_pose &b = g.poses[2 * f], &e = g.poses[2 * f + 1];
                qb = Q4{b.quat[0], b.quat[1], b.quat[2], b.quat[3]};
                qe = Q4{e.quat[0], e.quat[1], e.quat[2], e.quat[3]};
                tb = V3{b.tr[0], b.tr[1], b.tr[2]};
                te = V3{e.tr[0], e.tr[1], e.tr[2]};
                tsb = b.dest_timestamp;
                tse = e.dest_timestamp;
                sc = slerp_consts(qb, qe);
            }
#pragma unroll
            for (int k = 0; k < kPerThread; ++k) {
                const uint64_t i = c * kTile + (uint64_t) threadIdx.x * kPerThread + k;
                if (i >= g.n) break;
                const V3 w = random_point(P, pkey, i);
                if (!g.frames) {
                    pts[k] = w;
                    ts[k] = 0.0;
                    keep |= 1u << k;
                    continue;
                }
                const double alpha = (double) draw(pkey, i, 4) / kRandMax;
                ts[k] = tsb * (1.0 - alpha) + alpha * tse;
                // InterpolatePoseAlpha(begin, end, alpha).pose.Inverse() * world
                const Se3 inv = se3_inverse(Se3{qslerp_c(qb, qe, alpha, sc), (1.0 - alpha) * tb + alpha * te});
                const V3 raw = qrot(qnormalized(inv.q), w) + inv.t;
                if (norm3(raw.x, raw.y, raw.z) < g.d) {
                    pts[k] = sink.world ? w : raw;
                    keep |= 1u << k;
                }
            }
        }
        // block scan of the per-thread counts: thread order is point order
        const uint32_t cnt = __popc(keep);
        uint32_t incl = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        uint32_t before = incl - cnt, total = 0;
        for (int w = 0; w < kThreads / 32; ++w) {
            const uint32_t v = s_warp[w];
            if (w < warp) before += v;
            total += v;
        }
        if (warp == 0) {
            const uint32_t base = tile_lookback(g.desc, (int) tile, total);
            if (lane == 0) s_base = base;
        }
        __syncthreads();
        const uint64_t base = s_base;
        uint32_t pos = 0;
#pragma unroll
        for (int k = 0; k < kPerThread; ++k) {
            if (!((keep >> k) & 1u)) continue;
            const uint64_t out = base + before + pos++;
            if (out < sink.cap) {
                if (sink.data) store_gen_record(sink, out, pts[k], ts[k]);
                if (g.src) {
                    g.src[2 * out] = p;
                    g.src[2 * out + 1] = (uint32_t) (c * kTile + (uint64_t) threadIdx.x * kPerThread + k);
                }
            }
        }
        if (threadIdx.x == 0 && p == g.np - 1 && c == g.chunks - 1) g.ends[f] = base + total;
        __syncthreads();   // s_tile, s_warp and s_base are rewritten by the next tile
    }
}

// a grid-stride launch of n threads: at most 8 CTAs of kThreads per SM of the device
int Blocks(uint64_t n, int sms) {
    return (int) std::max<uint64_t>(1, std::min<uint64_t>((n + kThreads - 1) / kThreads, (uint64_t) sms * 8));
}

void CheckFinite(const double *v, uint64_t n, const char *what) {
    for (uint64_t i = 0; i < n; ++i)
        if (!std::isfinite(v[i])) throw std::invalid_argument(std::string(what) + ": a value is not finite");
}

void CheckDistance(double d) {
    if (!std::isfinite(d) || !(d > 0.0)) throw std::invalid_argument("distance must be finite and > 0");
}

}  // namespace

// ---- ColPivHouseholderQR<Matrix3d>::computeInPlace (Eigen 3.3.4+ / 3.4), host fp64 --------------------------------------
void FactorTriangle(SynPrim &t) {
    double (&a)[3][3] = t.qr;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) a[r][c] = t.p[c][r];   // A = [p0 p1 p2]
    const double eps = std::numeric_limits<double>::epsilon();
    double upd[3], direct[3];
    for (int k = 0; k < 3; ++k) upd[k] = direct[k] = norm3(a[0][k], a[1][k], a[2][k]);
    double maxn = upd[0];
    for (int k = 1; k < 3; ++k)
        if (upd[k] > maxn) maxn = upd[k];
    const double th = (maxn * eps) * (maxn * eps) / 3.0;
    const double downdate = std::sqrt(eps);
    int nonzero = 3, trans[3];
    for (int k = 0; k < 3; ++k) {
        int big = k;   // maxCoeff: the first largest
        for (int j = k + 1; j < 3; ++j)
            if (upd[j] > upd[big]) big = j;
        const double big_sq = upd[big] * upd[big];
        if (nonzero == 3 && big_sq < th * (double) (3 - k)) nonzero = k;
        trans[k] = big;
        if (big != k) {
            for (int r = 0; r < 3; ++r) std::swap(a[r][k], a[r][big]);
            std::swap(upd[k], upd[big]);
            std::swap(direct[k], direct[big]);
        }
        // makeHouseholderInPlace of a[k.., k]
        double tail = 0.0;
        for (int r = k + 1; r < 3; ++r) tail = r == k + 1 ? a[r][k] * a[r][k] : tail + a[r][k] * a[r][k];
        const double c0 = a[k][k];
        double beta, tau;
        if (tail <= std::numeric_limits<double>::min()) {
            tau = 0.0;
            beta = c0;
            for (int r = k + 1; r < 3; ++r) a[r][k] = 0.0;
        } else {
            beta = std::sqrt(c0 * c0 + tail);
            if (c0 >= 0.0) beta = -beta;
            for (int r = k + 1; r < 3; ++r) a[r][k] = a[r][k] / (c0 - beta);
            tau = (beta - c0) / beta;
        }
        t.tau[k] = tau;
        a[k][k] = beta;
        // applyHouseholderOnTheLeft to the columns after k
        if (k < 2 && tau != 0.0) {
            for (int j = k + 1; j < 3; ++j) {
                double tmp = a[k + 1][k] * a[k + 1][j];
                if (k == 0) tmp = tmp + a[2][0] * a[2][j];
                tmp += a[k][j];
                a[k][j] -= tau * tmp;
                for (int r = k + 1; r < 3; ++r) a[r][j] -= (tau * a[r][k]) * tmp;
            }
        }
        // the column norm downdate
        for (int j = k + 1; j < 3; ++j) {
            if (upd[j] != 0.0) {
                double tmp = std::fabs(a[k][j]) / upd[j];
                tmp = (1.0 + tmp) * (1.0 - tmp);
                tmp = tmp < 0.0 ? 0.0 : tmp;
                const double ratio = upd[j] / direct[j];
                const double tmp2 = tmp * (ratio * ratio);
                if (tmp2 <= downdate) {
                    double s = 0.0;
                    for (int r = k + 1; r < 3; ++r) s = r == k + 1 ? a[r][j] * a[r][j] : s + a[r][j] * a[r][j];
                    direct[j] = std::sqrt(s);
                    upd[j] = direct[j];
                } else {
                    upd[j] *= std::sqrt(tmp);
                }
            }
        }
    }
    t.rank = nonzero;
    int perm[3] = {0, 1, 2};
    for (int k = 0; k < 3; ++k) std::swap(perm[k], perm[trans[k]]);
    for (int k = 0; k < 3; ++k) t.perm[k] = perm[k];
}

SyntheticScene::SyntheticScene(const double *tri, uint64_t nt, const double *lines, uint64_t nl, const double *spheres,
                               uint64_t ns, const double *balls, uint64_t nb, int device)
    : device_(device) {
    if ((nt && !tri) || (nl && !lines) || (ns && !spheres) || (nb && !balls)) throw std::invalid_argument("null primitives");
    if (nt + nl + ns + nb > 0xFFFFFFFFull) throw std::invalid_argument("too many primitives");
    CheckFinite(tri, 9 * nt, "triangles");
    CheckFinite(lines, 6 * nl, "lines");
    CheckFinite(spheres, 4 * ns, "spheres");
    CheckFinite(balls, 4 * nb, "balls");
    for (uint64_t i = 0; i < ns; ++i)
        if (spheres[4 * i + 3] < 0.0) throw std::invalid_argument("spheres: a radius is negative");
    for (uint64_t i = 0; i < nb; ++i)
        if (balls[4 * i + 3] < 0.0) throw std::invalid_argument("balls: a radius is negative");
    prims_.reserve(nt + nl + ns + nb);
    for (uint64_t i = 0; i < nt; ++i) {
        SynPrim t{};
        t.kind = CTICP_SYN_TRIANGLE;
        for (int k = 0; k < 9; ++k) t.p[k / 3][k % 3] = tri[9 * i + k];
        // Normal(): (p0 - p2) x (p1 - p2), normalized (a zero vector stays zero)
        const double u[3] = {t.p[0][0] - t.p[2][0], t.p[0][1] - t.p[2][1], t.p[0][2] - t.p[2][2]};
        const double v[3] = {t.p[1][0] - t.p[2][0], t.p[1][1] - t.p[2][1], t.p[1][2] - t.p[2][2]};
        double n[3] = {u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0]};
        const double z = n[0] * n[0] + n[1] * n[1] + n[2] * n[2];
        if (z > 0.0)
            for (double &c : n) c /= std::sqrt(z);
        for (int k = 0; k < 3; ++k) {
            t.n[k] = n[k];
            t.b[k] = (t.p[0][k] + t.p[1][k] + t.p[2][k]) / 3.0;
        }
        FactorTriangle(t);
        prims_.push_back(t);
    }
    for (uint64_t i = 0; i < nl; ++i) {
        SynPrim l{};
        l.kind = CTICP_SYN_LINE;
        for (int k = 0; k < 6; ++k) l.p[k / 3][k % 3] = lines[6 * i + k];
        double d[3] = {l.p[0][0] - l.p[1][0], l.p[0][1] - l.p[1][1], l.p[0][2] - l.p[1][2]};
        const double z = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
        if (z > 0.0)
            for (double &c : d) c /= std::sqrt(z);
        for (int k = 0; k < 3; ++k) {
            l.n[k] = d[k];
            l.b[k] = (l.p[0][k] + l.p[1][k]) / 2.0;
        }
        prims_.push_back(l);
    }
    auto round = [&](const double *v, uint64_t n, int kind) {
        for (uint64_t i = 0; i < n; ++i) {
            SynPrim s{};
            s.kind = kind;
            for (int k = 0; k < 3; ++k) s.p[0][k] = v[4 * i + k];
            s.radius = v[4 * i + 3];
            prims_.push_back(s);
        }
    };
    round(spheres, ns, CTICP_SYN_SPHERE);
    round(balls, nb, CTICP_SYN_BALL);
    CT_CUDA_CHECK(cudaSetDevice(device_));
    CT_CUDA_CHECK(cudaDeviceGetAttribute(&sms_, cudaDevAttrMultiProcessorCount, device_));
    CT_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&generate_ctas_per_sm_, k_generate, kThreads, 0));
    generate_ctas_per_sm_ = std::max(generate_ctas_per_sm_, 1);
    stream_ = cticp::Stream(cudaStreamNonBlocking);
    ev_in_ = Event(cudaEventDisableTiming);
    ev_traj_ = Event(cudaEventDisableTiming);
    ev_out_ = Event(cudaEventDisableTiming);
    if (!prims_.empty()) {
        d_prims_.reserve(prims_.size(), stream_.get());
        CT_CUDA_CHECK(cudaMemcpyAsync(d_prims_.data(), prims_.data(), sizeof(SynPrim) * prims_.size(),
                                      cudaMemcpyHostToDevice, stream_.get()));
        CT_CUDA_CHECK(cudaStreamSynchronize(stream_.get()));
    }
}

SyntheticScene::~SyntheticScene() {
    if (stream_.get()) {
        cudaSetDevice(device_);
        cudaStreamSynchronize(stream_.get());
    }
}

void SyntheticScene::Distance(const double *points, uint64_t m, double *out) {
    if (m == 0 || prims_.empty()) return;
    if (!points || !out) throw std::invalid_argument("null argument");
    CT_CUDA_CHECK(cudaSetDevice(device_));
    cudaStream_t s = stream_.get();
    const uint64_t np = prims_.size();
    d_q_.reserve(3 * m, s);
    d_dist_.reserve(m * np, s);
    CT_CUDA_CHECK(cudaMemcpyAsync(d_q_.data(), points, sizeof(double) * 3 * m, cudaMemcpyHostToDevice, s));
    k_distance<<<Blocks(m * np, sms_), kThreads, 0, s>>>(d_prims_.data(), (uint32_t) np, d_q_.data(), m, d_dist_.data());
    CT_CUDA_CHECK(cudaGetLastError());
    CT_CUDA_CHECK(cudaMemcpyAsync(out, d_dist_.data(), sizeof(double) * m * np, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
}

void SyntheticScene::Launch(int mode, const Plan &plan, double distance, const double *location, uint64_t seed,
                            const cticp_synthetic_frame *frames, unsigned char *sink_data, const cticp_cloud_sink &sink,
                            uint64_t sink_cap, uint32_t *src_index, uint64_t *frame_ends) {
    cudaStream_t s = stream_.get();
    const uint64_t np = prims_.size();
    if (plan.tiles == 0) {   // no primitive: every frame is empty
        CT_CUDA_CHECK(cudaMemsetAsync(frame_ends, 0, sizeof(uint64_t) * plan.m, s));
        return;
    }
    d_sel_.reserve(plan.m * np, s);
    d_desc_.reserve(plan.tiles + 1, s);
    CT_CUDA_CHECK(cudaMemsetAsync(d_desc_.data(), 0, sizeof(unsigned long long) * (plan.tiles + 1), s));
    const double3 loc = location ? make_double3(location[0], location[1], location[2]) : make_double3(0, 0, 0);
    k_select<<<Blocks(plan.m * np, sms_), kThreads, 0, s>>>(d_prims_.data(), (uint32_t) np, plan.m, mode, d_poses_.data(), loc,
                                                      distance, d_sel_.data());
    CT_CUDA_CHECK(cudaGetLastError());
    GenArgs g{};
    g.prims = d_prims_.data();
    g.np = (uint32_t) np;
    g.n = plan.n;
    g.chunks = (plan.n + kTile - 1) / kTile;
    g.tiles = plan.tiles;
    g.sel = d_sel_.data();
    g.poses = d_poses_.data();
    g.frames = mode == 0 ? frames : nullptr;
    g.seed = seed;
    g.d = distance;
    g.desc = d_desc_.data();
    g.src = src_index;
    g.ends = frame_ends;
    // as many CTAs as are resident at once (tiles are handed out by the ticket, so any grid size is correct)
    const int blocks = (int) std::min<uint64_t>(plan.tiles, (uint64_t) sms_ * generate_ctas_per_sm_);
    k_generate<<<blocks, kThreads, 0, s>>>(g, MakeGenSink(sink_data, sink, sink_cap));
    CT_CUDA_CHECK(cudaGetLastError());
}

int64_t SyntheticScene::GeneratePoints(uint64_t n, const double *location, double distance, uint64_t seed, double *xyz,
                                       uint64_t cap, uint32_t *src_index) {
    if (location) {
        CheckFinite(location, 3, "location");
        if (std::isnan(distance)) throw std::invalid_argument("distance is NaN");
    }
    const uint64_t np = prims_.size();
    if (np && n > kMaxCandidates / np) throw CapacityError("more than 2^32 - 1 candidate points in one call");
    Plan plan{1, n, n ? np * ((n + kTile - 1) / kTile) : 0, n * np};
    if (n == 0) return 0;
    cticp_cloud_sink sink{};
    sink.point_step = 24;
    sink.xyz_dtype = CTICP_DTYPE_FLOAT64;
    sink.world = 1;
    const uint64_t m = std::min(cap, plan.upper);
    CT_CUDA_CHECK(cudaSetDevice(device_));
    cudaStream_t s = stream_.get();
    d_out_.reserve(std::max<uint64_t>(24 * m, 1), s);
    d_src_.reserve(std::max<uint64_t>(2 * m, 1), s);
    d_ends_.reserve(1, s);
    Launch(location ? 2 : 1, plan, distance, location, seed, nullptr, xyz ? d_out_.data() : nullptr, sink, m,
           src_index ? d_src_.data() : nullptr, d_ends_.data());
    uint64_t count = 0;
    CT_CUDA_CHECK(cudaMemcpyAsync(&count, d_ends_.data(), sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    const uint64_t w = std::min(cap, count);
    if (w && xyz) CT_CUDA_CHECK(cudaMemcpyAsync(xyz, d_out_.data(), 24 * w, cudaMemcpyDeviceToHost, s));
    if (w && src_index)
        CT_CUDA_CHECK(cudaMemcpyAsync(src_index, d_src_.data(), sizeof(uint32_t) * 2 * w, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    return (int64_t) count;
}

SyntheticScene::Plan SyntheticScene::CheckFrames(const ContinuousTrajectory &traj, const cticp_synthetic_frame *frames,
                                                 uint64_t m, uint64_t n, double distance,
                                                 const cticp_cloud_sink &sink) const {
    if (m && !frames) throw std::invalid_argument("null frames");
    if (traj.Device() != device_) throw std::invalid_argument("the trajectory lives on another device");
    CheckDistance(distance);
    if (n < 2) throw std::invalid_argument("Need to generate at least two points (num_points_per_primitive < 2)");
    for (uint64_t k = 0; k < m; ++k) {
        if (!std::isfinite(frames[k].begin_ts) || !std::isfinite(frames[k].end_ts))
            throw std::invalid_argument("frame " + std::to_string(k) + ": a timestamp is not finite");
        if (frames[k].begin_ts > frames[k].end_ts)
            throw std::invalid_argument("frame " + std::to_string(k) + ": begin_ts > end_ts");
    }
    CheckSink(sink);
    const uint64_t np = prims_.size();
    if (m && np && n > kMaxCandidates / np / m) throw CapacityError("more than 2^32 - 1 candidate points in one call");
    return Plan{m, n, m * np * ((n + kTile - 1) / kTile), m * np * n};
}

void SyntheticScene::Poses(ContinuousTrajectory &traj, const cticp_synthetic_frame *frames, uint64_t m) {
    cudaStream_t s = stream_.get();
    std::vector<double> ts(2 * m);
    for (uint64_t k = 0; k < m; ++k) {
        ts[2 * k] = frames[k].begin_ts;
        ts[2 * k + 1] = frames[k].end_ts;
    }
    d_q_.reserve(2 * m, s);
    d_poses_.reserve(2 * m, s);
    d_frames_.reserve(m, s);
    CT_CUDA_CHECK(cudaMemcpyAsync(d_q_.data(), ts.data(), sizeof(double) * 2 * m, cudaMemcpyHostToDevice, s));
    CT_CUDA_CHECK(cudaMemcpyAsync(d_frames_.data(), frames, sizeof(cticp_synthetic_frame) * m, cudaMemcpyHostToDevice, s));
    // the trajectory's kernel runs on its own stream, between two events of this one
    CT_CUDA_CHECK(cudaEventRecord(ev_traj_.get(), s));
    CT_CUDA_CHECK(cudaStreamWaitEvent(traj.Stream(), ev_traj_.get(), 0));
    traj.InterpolateDevice(d_q_.data(), 2 * m, d_poses_.data());
    CT_CUDA_CHECK(cudaEventRecord(ev_traj_.get(), traj.Stream()));
    CT_CUDA_CHECK(cudaStreamWaitEvent(s, ev_traj_.get(), 0));
    // the pageable copies above return once `ts` is staged; `ts` may go out of scope
}

int64_t SyntheticScene::GenerateFrames(ContinuousTrajectory &traj, const cticp_synthetic_frame *frames, uint64_t m,
                                       uint64_t n, double distance, uint64_t seed, const cticp_cloud_sink &sink,
                                       uint32_t *src_index, uint64_t *frame_ends) {
    if (m && !frame_ends) throw std::invalid_argument("null frame_ends");
    const Plan plan = CheckFrames(traj, frames, m, n, distance, sink);
    if (m == 0) return 0;
    const uint64_t cap = std::min<uint64_t>(sink.data || src_index ? sink.capacity_points : 0, plan.upper);
    const uint64_t out_bytes = sink.data && cap ? SpanBytes(cap, sink.point_step, SinkRecordWidth(sink), "sink") : 0;
    CT_CUDA_CHECK(cudaSetDevice(device_));
    cudaStream_t s = stream_.get();
    d_out_.reserve(std::max<uint64_t>(out_bytes, 1), s);
    d_src_.reserve(std::max<uint64_t>(2 * cap, 1), s);
    d_ends_.reserve(m, s);
    // the sink goes over as it is: its bytes outside x, y, z and t stay the caller's
    if (out_bytes) CT_CUDA_CHECK(cudaMemcpyAsync(d_out_.data(), sink.data, out_bytes, cudaMemcpyHostToDevice, s));
    Poses(traj, frames, m);
    Launch(0, plan, distance, nullptr, seed, d_frames_.data(), out_bytes ? d_out_.data() : nullptr, sink, cap,
           src_index ? d_src_.data() : nullptr, d_ends_.data());
    CT_CUDA_CHECK(cudaMemcpyAsync(frame_ends, d_ends_.data(), sizeof(uint64_t) * m, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    const uint64_t count = frame_ends[m - 1], w = std::min(cap, count);
    if (w && out_bytes)
        CT_CUDA_CHECK(cudaMemcpyAsync(sink.data, d_out_.data(), SpanBytes(w, sink.point_step, SinkRecordWidth(sink), "sink"),
                                      cudaMemcpyDeviceToHost, s));
    if (w && src_index)
        CT_CUDA_CHECK(cudaMemcpyAsync(src_index, d_src_.data(), sizeof(uint32_t) * 2 * w, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    return (int64_t) count;
}

void SyntheticScene::GenerateFramesDevice(ContinuousTrajectory &traj, const cticp_synthetic_frame *frames, uint64_t m,
                                          uint64_t n, double distance, uint64_t seed, const cticp_cloud_sink &sink,
                                          uint32_t *src_index, uint64_t *frame_ends, cudaStream_t stream) {
    if (m && !frame_ends) throw std::invalid_argument("null frame_ends");
    const Plan plan = CheckFrames(traj, frames, m, n, distance, sink);
    if (m == 0) return;
    const uint64_t cap = std::min<uint64_t>(sink.data || src_index ? sink.capacity_points : 0, plan.upper);
    CT_CUDA_CHECK(cudaSetDevice(device_));
    if (reinterpret_cast<uintptr_t>(frame_ends) % 8) throw std::invalid_argument("frame_ends is not 8-byte aligned");
    RequireDeviceRange(frame_ends, sizeof(uint64_t) * m, device_, "frame_ends");
    if (src_index && cap) {
        if (reinterpret_cast<uintptr_t>(src_index) % 4) throw std::invalid_argument("src_index is not 4-byte aligned");
        RequireDeviceRange(src_index, sizeof(uint32_t) * 2 * cap, device_, "src_index");
    }
    if (sink.data && cap)
        RequireDeviceRange(sink.data, SpanBytes(cap, sink.point_step, SinkRecordWidth(sink), "sink"), device_, "sink");
    cudaStream_t s = stream_.get();
    // ordered both ways with the caller's stream: behind what it queued before, ahead of what it queues next
    CT_CUDA_CHECK(cudaEventRecord(ev_in_.get(), stream));
    CT_CUDA_CHECK(cudaStreamWaitEvent(s, ev_in_.get(), 0));
    Poses(traj, frames, m);
    Launch(0, plan, distance, nullptr, seed, d_frames_.data(), sink.data && cap ? static_cast<unsigned char *>(sink.data) : nullptr,
           sink, cap, src_index && cap ? src_index : nullptr, frame_ends);
    CT_CUDA_CHECK(cudaEventRecord(ev_out_.get(), s));
    CT_CUDA_CHECK(cudaStreamWaitEvent(stream, ev_out_.get(), 0));
}

int64_t GeneratePoses(ContinuousTrajectory &traj, double frequency, cticp_pose *out, uint64_t cap) {
    if (cap && !out) throw std::invalid_argument("null out");
    if (!std::isfinite(frequency) || !(frequency > 0.0)) throw std::invalid_argument("frequency must be finite and > 0");
    const double step = 1.0 / frequency;
    double t = traj.MinTimestamp();
    const double max_t = traj.MaxTimestamp();
    if (!(max_t - t > step))
        throw std::invalid_argument("The interval between the first and last poses is too small for the frequency");
    std::vector<double> ts;
    while (t <= max_t) {
        if (ts.size() >= (1ull << 31)) throw std::invalid_argument("more than 2^31 poses");
        ts.push_back(t);
        t += step;
    }
    std::vector<cticp_pose> poses(ts.size());
    traj.Interpolate(ts.data(), nullptr, ts.size(), poses.data());
    std::copy(poses.begin(), poses.begin() + std::min<uint64_t>(cap, poses.size()), out);
    return (int64_t) poses.size();
}

void ApplyUniformNoise(cticp_pose *poses, uint64_t n, double scale_rot_deg, double scale_trans_m, uint64_t seed) {
    if (!std::isfinite(scale_rot_deg) || !std::isfinite(scale_trans_m)) throw std::invalid_argument("scales must be finite");
    for (uint64_t i = 0; i < n; ++i) {
        const uint64_t key = prim_key(seed, kKeyNoise, i);
        double r[6];
        for (uint32_t j = 0; j < 6; ++j) r[j] = rnd(draw(key, 0, j));
        // Random() * scale_rot_deg * M_PI / 180.0, then Random() * scale_trans_m
        double a[3];
        for (int j = 0; j < 3; ++j) a[j] = r[j] * scale_rot_deg * M_PI / 180.0;
        // Quaternion(AngleAxis): w = cos(angle / 2), vec = sin(angle / 2) axis; the three products in order
        Q4 q[3];
        for (int j = 0; j < 3; ++j) {
            const double ha = 0.5 * a[j], s = std::sin(ha);
            q[j] = Q4{s * (j == 0 ? 1.0 : 0.0), s * (j == 1 ? 1.0 : 0.0), s * (j == 2 ? 1.0 : 0.0), std::cos(ha)};
        }
        const Q4 qn = qnormalized(qnormalized(qmul(qmul(q[0], q[1]), q[2])));   // quat.normalized(), then SE3's own
        const Se3 noise{qn, V3{r[3] * scale_trans_m, r[4] * scale_trans_m, r[5] * scale_trans_m}};
        cticp_pose &p = poses[i];
        const Se3 out = se3_mul(noise, Se3{Q4{p.quat[0], p.quat[1], p.quat[2], p.quat[3]}, V3{p.tr[0], p.tr[1], p.tr[2]}});
        p.quat[0] = out.q.x; p.quat[1] = out.q.y; p.quat[2] = out.q.z; p.quat[3] = out.q.w;
        p.tr[0] = out.t.x; p.tr[1] = out.t.y; p.tr[2] = out.t.z;
    }
}

}  // namespace cticp
