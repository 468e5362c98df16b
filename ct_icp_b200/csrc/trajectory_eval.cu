// trajectory_eval.cu — kitti::EvaluatePoses and ComputeTrajectoryMetrics on the device.
//
// Reference: src/SlamCore/eval.cxx (ComputeMeanRPE :35-76, EvaluatePoses :103-111 and :136-178, ComputeTrajectoryMetrics
// :184-291), src/SlamCore/geometry.cxx:7-46 (OrthogonalProcrustes), include/SlamCore/types.h:326-350 (TSE3::Inverse,
// operator*) and :474-479 (TPose::Matrix).
//
// Per call, whatever the number of estimates B:
//   1. k_prep, one CTA, ground truth only: the distance steps in parallel, summed in index order by one thread with the
//      host's roundings (the pairs and the segment chain depend on every bit of them); then either the KITTI pairs (the
//      last frame of every (first frame, length) by a binary search, compacted in order) or the segment chain (one thread,
//      a binary search per segment).
//   2. KITTI: k_kitti, one CTA per estimate: APE, local error and the RPE of every kept pair.
//      Metrics: k_fit, one CTA per (segment, estimate) with the global fit as segment 0: centroids, cross-covariance,
//      a one-sided Jacobi SVD, the fitted transform and its errors; k_metrics_final, one thread per estimate.
// Every reduction is a fixed-order block reduction (no floating-point atomics): results are bit-reproducible and do not
// depend on which other estimates share the call.
#include "trajectory_eval.h"

#include <algorithm>
#include <cmath>
#include <limits>
#include <stdexcept>
#include <string>

#include "cuda_owner.h"
#include "se3.cuh"

namespace cticp {

namespace {

constexpr int kPrepThreads = 1024;
constexpr int kEvalThreads = 256;
constexpr uint32_t kStepSize = 10;   // the step_size EvaluatePoses passes to ComputeMeanRPE
constexpr int kPrepKitti = 0, kPrepChain = 1, kPrepDistances = 2;
constexpr int kDistKitti = 0, kDistTse3 = 1;

// ---- the distance steps with the host's roundings: no FMA contraction, the reference's operation order ---------------
__device__ __forceinline__ double norm_rn(double x, double y, double z) {
    return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
}
__device__ __forceinline__ V3 cross_rn(V3 a, V3 b) {
    return {__dsub_rn(__dmul_rn(a.y, b.z), __dmul_rn(a.z, b.y)), __dsub_rn(__dmul_rn(a.z, b.x), __dmul_rn(a.x, b.z)),
            __dsub_rn(__dmul_rn(a.x, b.y), __dmul_rn(a.y, b.x))};
}
// Eigen _transformVector (se3.cuh qrot) rounded step by step
__device__ __forceinline__ V3 qrot_rn(Q4 q, V3 v) {
    const V3 qv{q.x, q.y, q.z};
    V3 uv = cross_rn(qv, v);
    uv = {__dadd_rn(uv.x, uv.x), __dadd_rn(uv.y, uv.y), __dadd_rn(uv.z, uv.z)};
    const V3 c = cross_rn(qv, uv);
    return {__dadd_rn(__dadd_rn(v.x, __dmul_rn(q.w, uv.x)), c.x), __dadd_rn(__dadd_rn(v.y, __dmul_rn(q.w, uv.y)), c.y),
            __dadd_rn(__dadd_rn(v.z, __dmul_rn(q.w, uv.z)), c.z)};
}
__device__ __forceinline__ double qnorm2_rn(Q4 q) {
    return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(q.x, q.x), __dmul_rn(q.y, q.y)), __dmul_rn(q.z, q.z)), __dmul_rn(q.w, q.w));
}
__device__ __forceinline__ Q4 quat_of(const cticp_pose &p) { return Q4{p.quat[0], p.quat[1], p.quat[2], p.quat[3]}; }
__device__ __forceinline__ V3 tr_of(const cticp_pose &p) { return V3{p.tr[0], p.tr[1], p.tr[2]}; }

// step i >= 1 of kitti's trajectory_distances: |(poses[i-1] - poses[i]).t|
__device__ __forceinline__ double kitti_step(const cticp_pose &a, const cticp_pose &b) {
    return norm_rn(__dsub_rn(a.tr[0], b.tr[0]), __dsub_rn(a.tr[1], b.tr[1]), __dsub_rn(a.tr[2], b.tr[2]));
}
// step i >= 1 of ComputeTrajectoryMetrics: |(a.Inverse() * b).tr| in TSE3 arithmetic (quat.inverse(), then the product
// with quat.normalized())
__device__ __forceinline__ double tse3_step(const cticp_pose &a, const cticp_pose &b) {
    const Q4 q = quat_of(a);
    const double n2 = qnorm2_rn(q);
    const Q4 qi = n2 > 0 ? Q4{__ddiv_rn(-q.x, n2), __ddiv_rn(-q.y, n2), __ddiv_rn(-q.z, n2), __ddiv_rn(q.w, n2)}
                         : Q4{0, 0, 0, 0};
    const V3 ti = qrot_rn(qi, tr_of(a));
    const double ni = __dsqrt_rn(qnorm2_rn(qi));
    const Q4 qn{__ddiv_rn(qi.x, ni), __ddiv_rn(qi.y, ni), __ddiv_rn(qi.z, ni), __ddiv_rn(qi.w, ni)};
    const V3 r = qrot_rn(qn, tr_of(b));
    return norm_rn(__dsub_rn(r.x, ti.x), __dsub_rn(r.y, ti.y), __dsub_rn(r.z, ti.z));   // r + (-ti)
}

// a counted segment of the chain: poses [start, end], its length dist[end] - dist[start]
struct SegSpan {
    double length;
    int32_t start, end;
};

struct PrepArgs {
    const cticp_pose *gt;
    uint32_t n;
    int task, kind;
    double *dist;
    // KITTI pairs
    const double *lengths;
    uint32_t num_lengths;
    int32_t *last, *pos;   // per (first frame, length): the last frame (-1: skipped), the index among the kept pairs
    // segment chain
    double segment_length;
    SegSpan *spans;
    uint32_t max_spans;
    long long *count;      // kept pairs / counted segments
};

__global__ void __launch_bounds__(kPrepThreads) k_prep(PrepArgs a) {
    __shared__ double s_step[kPrepThreads];
    __shared__ int s_scan[kPrepThreads];
    __shared__ double s_run;
    __shared__ int s_base;
    const int tid = threadIdx.x;
    const uint32_t n = a.n;
    if (tid == 0) {
        s_run = 0.0;
        s_base = 0;
        a.dist[0] = 0.0;
    }
    __syncthreads();
    for (uint32_t base = 1; base < n; base += kPrepThreads) {
        const uint32_t i = base + tid;
        if (i < n) s_step[tid] = a.kind == kDistKitti ? kitti_step(a.gt[i - 1], a.gt[i]) : tse3_step(a.gt[i - 1], a.gt[i]);
        __syncthreads();
        if (tid == 0) {   // in index order: dist[i] = dist[i-1] + step[i]
            double d = s_run;
            const uint32_t m = min((uint32_t) kPrepThreads, n - base);
            for (uint32_t j = 0; j < m; ++j) {
                d = __dadd_rn(d, s_step[j]);
                a.dist[base + j] = d;
            }
            s_run = d;
        }
        __syncthreads();
    }
    const double *dist = a.dist;
    if (a.task == kPrepKitti) {
        const uint32_t L = a.num_lengths, F = (n + kStepSize - 1) / kStepSize, FL = F * L;
        for (uint32_t cb = 0; cb < FL; cb += kPrepThreads) {
            const uint32_t c = cb + tid;
            int flag = 0;
            if (c < FL) {
                // lastFrameFromSegmentLength: the first i >= first with dist[i] > dist[first] + len. dist does not
                // decrease, so the linear scan is an upper bound.
                const uint32_t first = (c / L) * kStepSize;
                const double v = dist[first] + a.lengths[c % L];
                uint32_t lo = first, hi = n;
                while (lo < hi) {
                    const uint32_t mid = (lo + hi) >> 1;
                    if (dist[mid] > v) hi = mid;
                    else lo = mid + 1;
                }
                flag = lo < n;
                a.last[c] = flag ? (int32_t) lo : -1;
            }
            s_scan[tid] = flag;   // inclusive scan over the CTA: the kept pairs stay in (first frame, length) order
            __syncthreads();
            for (int off = 1; off < kPrepThreads; off <<= 1) {
                const int v = tid >= off ? s_scan[tid - off] : 0;
                __syncthreads();
                s_scan[tid] += v;
                __syncthreads();
            }
            if (c < FL) a.pos[c] = flag ? s_base + s_scan[tid] - 1 : -1;
            __syncthreads();
            if (tid == 0) s_base += s_scan[kPrepThreads - 1];
            __syncthreads();
        }
        if (tid == 0) *a.count = s_base;
    } else if (a.task == kPrepChain && tid == 0) {
        // the greedy chain: the segment from `start` closes at the first idx with dist[idx] - last > segment_length
        // (monotone in idx, so a binary search); <= 5 poses: not counted, the chain still advances
        uint32_t start = 0, from = 0, k = 0;
        double last = 0.0;
        while (from < n) {
            uint32_t lo = from, hi = n;
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (__dsub_rn(dist[mid], last) > a.segment_length) hi = mid;
                else lo = mid + 1;
            }
            if (lo >= n) break;
            if (lo - start + 1 > 5 && k < a.max_spans) a.spans[k++] = SegSpan{__dsub_rn(dist[lo], last), (int32_t) start, (int32_t) lo};
            start = lo;
            last = dist[lo];
            from = lo + 1;
        }
        *a.count = k;
    }
}

// ---- fixed-order block reductions (blockDim.x = kEvalThreads, a power of two) -----------------------------------------
__device__ double block_sum(double v, double *sh) {
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int s = kEvalThreads / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
        __syncthreads();
    }
    const double r = sh[0];
    __syncthreads();
    return r;
}
__device__ double block_max(double v, double *sh) {
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int s = kEvalThreads / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s && sh[threadIdx.x] < sh[threadIdx.x + s]) sh[threadIdx.x] = sh[threadIdx.x + s];
        __syncthreads();
    }
    const double r = sh[0];
    __syncthreads();
    return r;
}
// the largest value and the first index holding it: the reference's running max with a strict comparison, where each
// thread's (v, i) is its own running max over increasing indices from the same start value
__device__ void block_argmax(double &v, long long &i, double *sh, long long *shi) {
    sh[threadIdx.x] = v;
    shi[threadIdx.x] = i;
    __syncthreads();
    for (int s = kEvalThreads / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) {
            const double o = sh[threadIdx.x + s];
            const long long oi = shi[threadIdx.x + s];
            if (o > sh[threadIdx.x] || (o == sh[threadIdx.x] && oi < shi[threadIdx.x])) {
                sh[threadIdx.x] = o;
                shi[threadIdx.x] = oi;
            }
        }
        __syncthreads();
    }
    v = sh[0];
    i = shi[0];
    __syncthreads();
}

// ---- KITTI: rigid 3×4 matrices of TPose::Matrix (quat.normalized().toRotationMatrix(), tr) ----------------------------
struct Rt {
    M3 R;
    V3 t;
};
__device__ __forceinline__ Rt matrix_of(const cticp_pose &p) { return Rt{qtoR(qnormalized(quat_of(p))), tr_of(p)}; }
__device__ __forceinline__ Rt rigid_inverse(const Rt &a) {   // the inverse of [R t; 0 1]: [R^T, -R^T t]
    Rt r;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) r.R.m[i][j] = a.R.m[j][i];
    const V3 v = {r.R.m[0][0] * a.t.x + r.R.m[0][1] * a.t.y + r.R.m[0][2] * a.t.z,
                  r.R.m[1][0] * a.t.x + r.R.m[1][1] * a.t.y + r.R.m[1][2] * a.t.z,
                  r.R.m[2][0] * a.t.x + r.R.m[2][1] * a.t.y + r.R.m[2][2] * a.t.z};
    r.t = {-v.x, -v.y, -v.z};
    return r;
}
__device__ __forceinline__ Rt rt_mul(const Rt &a, const Rt &b) {
    Rt r;
    r.R = mmul(a.R, b.R);
    r.t = {a.R.m[0][0] * b.t.x + a.R.m[0][1] * b.t.y + a.R.m[0][2] * b.t.z + a.t.x,
           a.R.m[1][0] * b.t.x + a.R.m[1][1] * b.t.y + a.R.m[1][2] * b.t.z + a.t.y,
           a.R.m[2][0] * b.t.x + a.R.m[2][1] * b.t.y + a.R.m[2][2] * b.t.z + a.t.z};
    return r;
}

struct KittiArgs {
    const cticp_pose *gt, *est;
    uint32_t n, num_lengths, num_candidates;   // candidates: (first frame, length) pairs, first-frame-major
    const double *lengths;
    const int32_t *last, *pos;
    const long long *count;
    double *tab;   // B × num_candidates × 2: the kept pairs of estimate b from tab[2 * b * num_candidates]
    cticp_kitti_errors *out;
};

__global__ void __launch_bounds__(kEvalThreads) k_kitti(KittiArgs a) {
    __shared__ double sh[kEvalThreads];
    __shared__ long long shi[kEvalThreads];
    const int b = blockIdx.x;
    const uint32_t n = a.n;
    const cticp_pose *gt = a.gt, *est = a.est + (size_t) b * n;
    double s_ape = 0.0, m_ape = 0.0, s_loc = 0.0, m_loc = 0.0, s_rpe = 0.0;
    long long i_loc = 0;
    for (uint32_t i = threadIdx.x; i < n; i += kEvalThreads) {
        const Rt e = matrix_of(est[i]);
        const V3 d = rt_mul(rigid_inverse(e), matrix_of(gt[i])).t;
        const double ape = norm(d);
        s_ape += ape;
        if (m_ape < ape) m_ape = ape;
        if (i >= 1) {
            const double loc = fabs(norm(tr_of(gt[i]) - tr_of(gt[i - 1])) - norm(tr_of(est[i]) - tr_of(est[i - 1])));
            s_loc += loc;
            if (m_loc < loc) {
                m_loc = loc;
                i_loc = i;
            }
        }
    }
    double *tab = a.tab + (size_t) 2 * b * a.num_candidates;
    for (uint32_t c = threadIdx.x; c < a.num_candidates; c += kEvalThreads) {
        const int32_t last = a.last[c];
        if (last < 0) continue;
        const uint32_t first = (c / a.num_lengths) * kStepSize;
        const double len = a.lengths[c % a.num_lengths];
        const Rt dg = rt_mul(rigid_inverse(matrix_of(gt[first])), matrix_of(gt[last]));
        const Rt de = rt_mul(rigid_inverse(matrix_of(est[first])), matrix_of(est[last]));
        const Rt E = rt_mul(rigid_inverse(de), dg);
        const double t_err = norm(E.t);
        const double d = 0.5 * (E.R.m[0][0] + E.R.m[1][1] + E.R.m[2][2] - 1.0);
        const double r_err = acos(fmax(fmin(d, 1.0), -1.0));
        const int32_t p = a.pos[c];
        tab[2 * p] = t_err / len;
        tab[2 * p + 1] = r_err / len;
        s_rpe += t_err / len;
    }
    s_ape = block_sum(s_ape, sh);
    s_loc = block_sum(s_loc, sh);
    s_rpe = block_sum(s_rpe, sh);
    m_ape = block_max(m_ape, sh);
    block_argmax(m_loc, i_loc, sh, shi);
    if (threadIdx.x == 0) {
        cticp_kitti_errors r;
        r.mean_rpe = (s_rpe / (double) *a.count) * 100.0;   // no pair: 0 / 0
        r.mean_ape = s_ape / (double) n;
        r.max_ape = m_ape;
        r.mean_local_err = s_loc / (double) (n - 1);       // n = 1: 0 / 0
        r.max_local_err = m_loc;
        r.index_max_local_err = i_loc;
        a.out[b] = r;
    }
}

// ---- OrthogonalProcrustes ------------------------------------------------------------------------------------------
// 3×3 SVD A = U diag(s) V^T by one-sided Jacobi (rotations of the columns of A until they are orthogonal), singular
// values in decreasing order as Eigen's JacobiSVD returns them. Rank deficiency: a column whose norm is zero (or below
// 1e-13 of the largest) takes the direction that completes U to a right-handed orthonormal basis; A = 0 gives U = V = I.
__device__ void svd3(const double Ain[3][3], double U[3][3], double V[3][3]) {
    double A[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            A[i][j] = Ain[i][j];
            V[i][j] = i == j ? 1.0 : 0.0;
        }
    const int P[3] = {0, 0, 1}, Q[3] = {1, 2, 2};
    for (int sweep = 0; sweep < 16; ++sweep) {
        bool rotated = false;
        for (int k = 0; k < 3; ++k) {
            const int p = P[k], q = Q[k];
            double al = 0, be = 0, ga = 0;
            for (int r = 0; r < 3; ++r) {
                al += A[r][p] * A[r][p];
                be += A[r][q] * A[r][q];
                ga += A[r][p] * A[r][q];
            }
            if (!(fabs(ga) > 1e-15 * sqrt(al) * sqrt(be))) continue;
            rotated = true;
            const double zeta = (be - al) / (2.0 * ga);
            const double t = fabs(zeta) > 1e150 ? 0.5 / zeta
                                                : (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
            const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
            for (int r = 0; r < 3; ++r) {
                const double ap = A[r][p], aq = A[r][q];
                A[r][p] = c * ap - s * aq;
                A[r][q] = s * ap + c * aq;
                const double vp = V[r][p], vq = V[r][q];
                V[r][p] = c * vp - s * vq;
                V[r][q] = s * vp + c * vq;
            }
        }
        if (!rotated) break;
    }
    double sv[3];
    for (int j = 0; j < 3; ++j) sv[j] = sqrt(A[0][j] * A[0][j] + A[1][j] * A[1][j] + A[2][j] * A[2][j]);
    auto swap_cols = [&](int i, int j) {
        const double t = sv[i]; sv[i] = sv[j]; sv[j] = t;
        for (int r = 0; r < 3; ++r) {
            double x = A[r][i]; A[r][i] = A[r][j]; A[r][j] = x;
            x = V[r][i]; V[r][i] = V[r][j]; V[r][j] = x;
        }
    };
    if (sv[1] > sv[0]) swap_cols(0, 1);
    if (sv[2] > sv[1]) swap_cols(1, 2);
    if (sv[1] > sv[0]) swap_cols(0, 1);
    if (!(sv[0] > 0.0)) {
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) U[i][j] = i == j ? 1.0 : 0.0;
        return;
    }
    const double tol = 1e-13 * sv[0];
    V3 u[3];
    u[0] = (1.0 / sv[0]) * V3{A[0][0], A[1][0], A[2][0]};
    if (sv[1] > tol) {
        u[1] = (1.0 / sv[1]) * V3{A[0][1], A[1][1], A[2][1]};
    } else {   // any unit vector orthogonal to u0: u0 × the axis it leans on least
        const double ax = fabs(u[0].x), ay = fabs(u[0].y), az = fabs(u[0].z);
        const V3 e = (ax <= ay && ax <= az) ? V3{1, 0, 0} : (ay <= az ? V3{0, 1, 0} : V3{0, 0, 1});
        const V3 w = cross(u[0], e);
        u[1] = (1.0 / norm(w)) * w;
    }
    u[2] = sv[2] > tol ? (1.0 / sv[2]) * V3{A[0][2], A[1][2], A[2][2]} : cross(u[0], u[1]);
    for (int j = 0; j < 3; ++j) {
        U[0][j] = u[j].x;
        U[1][j] = u[j].y;
        U[2][j] = u[j].z;
    }
}

// geometry.cxx:7-46 from the centroids and the cross-covariance M = sum (tgt - ct)(ref - cr)^T
__device__ Se3 procrustes(const double M[3][3], V3 cr, V3 ct) {
    double U[3][3], V[3][3];
    svd3(M, U, V);
    M3 R;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) R.m[i][j] = U[i][0] * V[j][0] + U[i][1] * V[j][1] + U[i][2] * V[j][2];
    const double det = R.m[0][0] * (R.m[1][1] * R.m[2][2] - R.m[1][2] * R.m[2][1]) -
                       R.m[0][1] * (R.m[1][0] * R.m[2][2] - R.m[1][2] * R.m[2][0]) +
                       R.m[0][2] * (R.m[1][0] * R.m[2][1] - R.m[1][1] * R.m[2][0]);
    if (det < 0.0)   // U diag(1, 1, -1) V^T
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) R.m[i][j] = U[i][0] * V[j][0] + U[i][1] * V[j][1] - U[i][2] * V[j][2];
    Se3 T;
    T.q = qnormalized(qfromR(R));
    T.t = ct - qrot(T.q, cr);
    return T;
}

struct FitArgs {
    const cticp_pose *gt, *est;
    uint32_t n, max_spans;
    const SegSpan *spans;
    const long long *count;
    cticp_traj_segment *segs;   // B × max_spans
    cticp_traj_metrics *out;    // B
};

// blockIdx.x = 0: the global fit over [0, n) and the ATE; blockIdx.x = k + 1: counted segment k; blockIdx.y: estimate
__global__ void __launch_bounds__(kEvalThreads) k_fit(FitArgs a) {
    __shared__ double sh[kEvalThreads];
    __shared__ long long shi[kEvalThreads];
    __shared__ Se3 s_T;
    const int b = blockIdx.y;
    const bool global = blockIdx.x == 0;
    uint32_t first = 0, m = a.n;
    if (!global) {
        const long long k = blockIdx.x - 1;
        if (k >= *a.count) return;   // uniform over the CTA
        first = (uint32_t) a.spans[k].start;
        m = (uint32_t) a.spans[k].end - first + 1;
    }
    const cticp_pose *G = a.gt + first, *E = a.est + (size_t) b * a.n + first;
    double c[6] = {0, 0, 0, 0, 0, 0};
    for (uint32_t i = threadIdx.x; i < m; i += kEvalThreads) {
        for (int k = 0; k < 3; ++k) {
            c[k] += G[i].tr[k];
            c[3 + k] += E[i].tr[k];
        }
    }
    for (int k = 0; k < 6; ++k) c[k] = block_sum(c[k], sh) / (double) m;
    const V3 cr{c[0], c[1], c[2]}, ct{c[3], c[4], c[5]};
    double M[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    for (uint32_t i = threadIdx.x; i < m; i += kEvalThreads) {
        const V3 dr = tr_of(G[i]) - cr, dt = tr_of(E[i]) - ct;
        const double r[3] = {dr.x, dr.y, dr.z}, t[3] = {dt.x, dt.y, dt.z};
        for (int p = 0; p < 3; ++p)
            for (int q = 0; q < 3; ++q) M[p][q] += t[p] * r[q];
    }
    for (int p = 0; p < 3; ++p)
        for (int q = 0; q < 3; ++q) M[p][q] = block_sum(M[p][q], sh);
    if (threadIdx.x == 0) s_T = procrustes(M, cr, ct);
    __syncthreads();
    const Se3 T = s_T;
    const Q4 qn = qnormalized(T.q);   // TSE3::operator* normalises the quaternion again
    double s = 0.0, mx = global ? 0.0 : -1.0;
    long long imx = -1;
    for (uint32_t i = threadIdx.x; i < m; i += kEvalThreads) {
        const double e = norm(qrot(qn, tr_of(G[i])) + T.t - tr_of(E[i]));
        s += e;
        if (e > mx) {
            mx = e;
            imx = i;
        }
    }
    if (global) {
        s = block_sum(s, sh);
        block_argmax(mx, imx, sh, shi);
        if (threadIdx.x == 0) {
            cticp_traj_metrics &r = a.out[b];
            r.mean_ate = s / (double) m;
            r.max_ate = mx;
            r.max_ate_idx = imx;
            r.quat[0] = T.q.x; r.quat[1] = T.q.y; r.quat[2] = T.q.z; r.quat[3] = T.q.w;
            r.tr[0] = T.t.x; r.tr[1] = T.t.y; r.tr[2] = T.t.z;
        }
    } else {
        mx = block_max(mx, sh);
        if (threadIdx.x == 0) {
            const SegSpan sp = a.spans[blockIdx.x - 1];
            cticp_traj_segment &r = a.segs[(size_t) b * a.max_spans + blockIdx.x - 1];
            r.segment_length = sp.length;
            r.start_idx = sp.start;
            r.end_idx = sp.end;
            r.loc_error = mx;
            r.quat[0] = T.q.x; r.quat[1] = T.q.y; r.quat[2] = T.q.z; r.quat[3] = T.q.w;
            r.tr[0] = T.t.x; r.tr[1] = T.t.y; r.tr[2] = T.t.z;
        }
    }
}

// the segment means of each estimate, summed in segment order as the reference does
__global__ void k_metrics_final(const double *dist, uint32_t n, const long long *count, const cticp_traj_segment *segs,
                                uint32_t max_spans, size_t num_estimates, cticp_traj_metrics *out) {
    const size_t b = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
    if (b >= num_estimates) return;
    const long long S = *count;
    double sr = 0.0, sl = 0.0;   // the reference leaves the ratio's accumulator uninitialised (eval.h:88)
    for (long long k = 0; k < S; ++k) {
        const cticp_traj_segment &s = segs[b * max_spans + k];
        sr += s.loc_error / s.segment_length;
        sl += s.loc_error;
    }
    cticp_traj_metrics &r = out[b];
    r.total_distance = dist[n - 1];
    r.segment_mean_ate_ratio = sr / (double) S;   // no counted segment: 0 / 0
    r.segment_mean_ate = sl / (double) S;
    r.num_segments = S;
}

// ---- host side -----------------------------------------------------------------------------------------------------
// one device allocation per call, carved into 256-byte aligned pieces
struct Arena {
    size_t bytes = 0;
    template <typename T>
    size_t add(size_t count) {
        const size_t off = bytes;
        bytes += (sizeof(T) * std::max<size_t>(count, 1) + 255) & ~size_t(255);
        return off;
    }
};
template <typename T>
T *at(const DeviceArray<unsigned char> &buf, size_t off) {
    return reinterpret_cast<T *>(buf.data() + off);
}

void CheckPoses(const cticp_pose *p, size_t count, bool timestamps, const char *what) {
    for (size_t i = 0; i < count; ++i) {
        const cticp_pose &q = p[i];
        double n2 = 0;
        bool finite = true;
        for (int k = 0; k < 4; ++k) {
            finite = finite && std::isfinite(q.quat[k]);
            n2 += q.quat[k] * q.quat[k];
        }
        if (!finite || !(n2 > 0) || !std::isfinite(n2))
            throw std::invalid_argument(std::string(what) + " pose " + std::to_string(i) +
                                        ": the quaternion must be finite and non-zero");
        for (int k = 0; k < 3; ++k)
            if (!std::isfinite(q.tr[k]))
                throw std::invalid_argument(std::string(what) + " pose " + std::to_string(i) + ": non-finite translation");
        if (timestamps && !std::isfinite(q.dest_timestamp))
            throw std::invalid_argument(std::string(what) + " pose " + std::to_string(i) + ": non-finite dest_timestamp");
    }
}

void CheckGroundTruth(const cticp_pose *gt, size_t n, size_t min_n) {
    if (!gt) throw std::invalid_argument("null ground truth");
    if (n < min_n)
        throw std::invalid_argument(min_n > 1 ? "Cannot estimate the trajectory metrics with less than 5 poses"
                                              : "no ground-truth poses");
    if (n > (size_t) std::numeric_limits<int32_t>::max()) throw std::invalid_argument("too many poses");
    CheckPoses(gt, n, true, "ground-truth");
}

void CheckEstimates(const cticp_pose *est, size_t n, size_t num_estimates) {
    if (!est) throw std::invalid_argument("null estimates");
    if (num_estimates == 0) throw std::invalid_argument("no estimates");
    if (num_estimates > std::numeric_limits<size_t>::max() / sizeof(cticp_pose) / n)
        throw std::invalid_argument("too many estimates");
    CheckPoses(est, n * num_estimates, false, "estimated");
}

void CheckLengths(const double *lengths, size_t num_lengths) {
    if (num_lengths == 0 || !lengths) throw std::invalid_argument("empty length list");
    if (num_lengths > 1024 * 1024) throw std::invalid_argument("too many lengths");
    for (size_t i = 0; i < num_lengths; ++i)
        if (!(std::isfinite(lengths[i]) && lengths[i] > 0))
            throw std::invalid_argument("lengths must be finite and > 0");
}

uint32_t NumCandidates(size_t n, size_t L) {
    const size_t fl = ((n + kStepSize - 1) / kStepSize) * L;
    if (fl > (size_t) std::numeric_limits<int32_t>::max()) throw std::invalid_argument("too many (first frame, length) pairs");
    return (uint32_t) fl;
}

// the device buffers of one KITTI evaluation of B estimates, carved from one allocation
struct KittiBuffers {
    DeviceArray<unsigned char> buf;
    PrepArgs prep{};
    KittiArgs eval{};
    double *ts = nullptr;   // the ground-truth timestamps (trajectory form only)

    KittiBuffers(size_t n, size_t B, size_t L, bool with_timestamps, cudaStream_t s) {
        const uint32_t FL = NumCandidates(n, L);
        Arena ar;
        const size_t o_gt = ar.add<cticp_pose>(n), o_est = ar.add<cticp_pose>(B * n), o_dist = ar.add<double>(n),
                     o_len = ar.add<double>(L), o_last = ar.add<int32_t>(FL), o_pos = ar.add<int32_t>(FL),
                     o_count = ar.add<long long>(1), o_tab = ar.add<double>(2 * (size_t) FL * B),
                     o_out = ar.add<cticp_kitti_errors>(B), o_ts = ar.add<double>(with_timestamps ? n : 0);
        buf.reserve(ar.bytes, s);
        prep.gt = at<cticp_pose>(buf, o_gt);
        prep.n = (uint32_t) n;
        prep.task = kPrepKitti;
        prep.kind = kDistKitti;
        prep.dist = at<double>(buf, o_dist);
        prep.lengths = at<double>(buf, o_len);
        prep.num_lengths = (uint32_t) L;
        prep.last = at<int32_t>(buf, o_last);
        prep.pos = at<int32_t>(buf, o_pos);
        prep.count = at<long long>(buf, o_count);
        eval.gt = prep.gt;
        eval.est = at<cticp_pose>(buf, o_est);
        eval.n = (uint32_t) n;
        eval.num_lengths = (uint32_t) L;
        eval.num_candidates = FL;
        eval.lengths = prep.lengths;
        eval.last = prep.last;
        eval.pos = prep.pos;
        eval.count = prep.count;
        eval.tab = at<double>(buf, o_tab);
        eval.out = at<cticp_kitti_errors>(buf, o_out);
        if (with_timestamps) ts = at<double>(buf, o_ts);
    }
    cticp_pose *Estimates() const { return const_cast<cticp_pose *>(eval.est); }
};

// the KITTI evaluation of the B estimates already in (or queued for) kb.eval.est against gt (host), on stream s
int64_t RunKitti(cudaStream_t s, KittiBuffers &kb, const cticp_pose *gt, size_t n, size_t B, const double *lengths,
                 size_t L, cticp_kitti_errors *out, double *tab_errors, size_t cap) {
    const PrepArgs &p = kb.prep;
    const KittiArgs &k = kb.eval;
    const uint32_t FL = k.num_candidates;
    CT_CUDA_CHECK(cudaMemcpyAsync(const_cast<cticp_pose *>(p.gt), gt, sizeof(cticp_pose) * n, cudaMemcpyHostToDevice, s));
    CT_CUDA_CHECK(cudaMemcpyAsync(const_cast<double *>(p.lengths), lengths, sizeof(double) * L, cudaMemcpyHostToDevice, s));
    k_prep<<<1, kPrepThreads, 0, s>>>(p);
    CT_CUDA_CHECK(cudaGetLastError());
    k_kitti<<<(unsigned) B, kEvalThreads, 0, s>>>(k);
    CT_CUDA_CHECK(cudaGetLastError());
    long long count = 0;
    CT_CUDA_CHECK(cudaMemcpyAsync(out, k.out, sizeof(cticp_kitti_errors) * B, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaMemcpyAsync(&count, p.count, sizeof(long long), cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    const size_t m = std::min<size_t>(cap, (size_t) count);
    if (tab_errors && m) {
        CT_CUDA_CHECK(cudaMemcpy2DAsync(tab_errors, 2 * sizeof(double) * cap, k.tab, 2 * sizeof(double) * FL,
                                        2 * sizeof(double) * m, B, cudaMemcpyDeviceToHost, s));
        CT_CUDA_CHECK(cudaStreamSynchronize(s));
    }
    return count;
}

}  // namespace

void CheckKittiArgs(const cticp_pose *gt, size_t n, const cticp_pose *est, size_t num_estimates, const double *lengths,
                    size_t num_lengths, const cticp_kitti_errors *out) {
    CheckKittiTrajectoryArgs(gt, n, lengths, num_lengths, out);
    CheckEstimates(est, n, num_estimates);
}

void CheckKittiTrajectoryArgs(const cticp_pose *gt, size_t n, const double *lengths, size_t num_lengths,
                              const cticp_kitti_errors *out) {
    if (!out) throw std::invalid_argument("null output");
    CheckGroundTruth(gt, n, 1);
    CheckLengths(lengths, num_lengths);
    NumCandidates(n, num_lengths);
}

void CheckMetricsArgs(const cticp_pose *gt, size_t n, const cticp_pose *est, size_t num_estimates,
                      double segment_length, const cticp_traj_metrics *out) {
    if (!out) throw std::invalid_argument("null output");
    if (!(std::isfinite(segment_length) && segment_length > 0))
        throw std::invalid_argument("segment_length must be finite and > 0");
    CheckGroundTruth(gt, n, 6);
    CheckEstimates(est, n, num_estimates);
}

void CheckDistancesArgs(const cticp_pose *gt, size_t n, int kind, const double *out) {
    if (!out) throw std::invalid_argument("null output");
    if (kind != kDistKitti && kind != kDistTse3) throw std::invalid_argument("kind must be 0 (KITTI) or 1 (metrics)");
    CheckGroundTruth(gt, n, 1);
}

int64_t KittiEvaluate(const cticp_pose *gt, size_t n, const cticp_pose *est, size_t B, const double *lengths, size_t L,
                      cticp_kitti_errors *out, double *tab_errors, size_t cap) {
    // a blocking stream: ordered with the legacy default stream, so events recorded there bracket the call
    const cticp::Stream stream(cudaStreamDefault);
    KittiBuffers kb(n, B, L, false, stream.get());
    CT_CUDA_CHECK(cudaMemcpyAsync(kb.Estimates(), est, sizeof(cticp_pose) * n * B, cudaMemcpyHostToDevice, stream.get()));
    return RunKitti(stream.get(), kb, gt, n, B, lengths, L, out, tab_errors, cap);
}

int64_t KittiEvaluateTrajectory(ContinuousTrajectory &t, const cticp_pose *gt, size_t n, const double *lengths,
                                size_t L, cticp_kitti_errors *out, double *tab_errors, size_t cap) {
    CT_CUDA_CHECK(cudaSetDevice(t.Device()));
    cudaStream_t s = t.Stream();
    KittiBuffers kb(n, 1, L, true, s);
    std::vector<double> ts(n);
    for (size_t i = 0; i < n; ++i) ts[i] = gt[i].dest_timestamp;
    CT_CUDA_CHECK(cudaMemcpyAsync(kb.ts, ts.data(), sizeof(double) * n, cudaMemcpyHostToDevice, s));
    // EvaluatePoses(gt, trajectory): est_i = InterpolatePose(gt_i.dest_timestamp, true), on the trajectory's stream
    t.InterpolateDevice(kb.ts, n, kb.Estimates());
    return RunKitti(s, kb, gt, n, 1, lengths, L, out, tab_errors, cap);
}

int64_t TrajectoryMetrics(const cticp_pose *gt, size_t n, const cticp_pose *est, size_t B, double segment_length,
                          cticp_traj_metrics *out, cticp_traj_segment *segments, size_t cap) {
    // a counted segment spans at least 5 steps and segments share only their end poses
    const uint32_t max_spans = (uint32_t) std::max<size_t>(1, (n - 1) / 5);
    Arena ar;
    const size_t o_gt = ar.add<cticp_pose>(n), o_est = ar.add<cticp_pose>(B * n), o_dist = ar.add<double>(n),
                 o_spans = ar.add<SegSpan>(max_spans), o_count = ar.add<long long>(1),
                 o_segs = ar.add<cticp_traj_segment>((size_t) max_spans * B), o_out = ar.add<cticp_traj_metrics>(B);
    const cticp::Stream stream(cudaStreamDefault);
    cudaStream_t s = stream.get();
    DeviceArray<unsigned char> buf;
    buf.reserve(ar.bytes, s);
    CT_CUDA_CHECK(cudaMemcpyAsync(at<cticp_pose>(buf, o_gt), gt, sizeof(cticp_pose) * n, cudaMemcpyHostToDevice, s));
    CT_CUDA_CHECK(cudaMemcpyAsync(at<cticp_pose>(buf, o_est), est, sizeof(cticp_pose) * n * B, cudaMemcpyHostToDevice, s));
    PrepArgs p{};
    p.gt = at<cticp_pose>(buf, o_gt);
    p.n = (uint32_t) n;
    p.task = kPrepChain;
    p.kind = kDistTse3;
    p.dist = at<double>(buf, o_dist);
    p.segment_length = segment_length;
    p.spans = at<SegSpan>(buf, o_spans);
    p.max_spans = max_spans;
    p.count = at<long long>(buf, o_count);
    k_prep<<<1, kPrepThreads, 0, s>>>(p);
    CT_CUDA_CHECK(cudaGetLastError());
    FitArgs f{};
    f.gt = p.gt;
    f.est = at<cticp_pose>(buf, o_est);
    f.n = (uint32_t) n;
    f.max_spans = max_spans;
    f.spans = p.spans;
    f.count = p.count;
    f.segs = at<cticp_traj_segment>(buf, o_segs);
    f.out = at<cticp_traj_metrics>(buf, o_out);
    for (size_t b0 = 0; b0 < B; b0 += 65535) {   // gridDim.y limit
        FitArgs fb = f;
        fb.est += b0 * n;
        fb.segs += b0 * max_spans;
        fb.out += b0;
        const unsigned nb = (unsigned) std::min<size_t>(B - b0, 65535);
        k_fit<<<dim3(1 + max_spans, nb), kEvalThreads, 0, s>>>(fb);
        CT_CUDA_CHECK(cudaGetLastError());
    }
    k_metrics_final<<<(unsigned) ((B + 127) / 128), 128, 0, s>>>(p.dist, (uint32_t) n, p.count, f.segs, max_spans, B, f.out);
    CT_CUDA_CHECK(cudaGetLastError());
    long long count = 0;
    CT_CUDA_CHECK(cudaMemcpyAsync(out, f.out, sizeof(cticp_traj_metrics) * B, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaMemcpyAsync(&count, p.count, sizeof(long long), cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    const size_t m = std::min<size_t>(cap, (size_t) count);
    if (segments && m) {
        CT_CUDA_CHECK(cudaMemcpy2DAsync(segments, sizeof(cticp_traj_segment) * cap, f.segs,
                                        sizeof(cticp_traj_segment) * max_spans, sizeof(cticp_traj_segment) * m, B,
                                        cudaMemcpyDeviceToHost, s));
        CT_CUDA_CHECK(cudaStreamSynchronize(s));
    }
    return count;
}

void TrajectoryDistances(const cticp_pose *gt, size_t n, int kind, double *out) {
    Arena ar;
    const size_t o_gt = ar.add<cticp_pose>(n), o_dist = ar.add<double>(n), o_count = ar.add<long long>(1);
    const cticp::Stream stream(cudaStreamDefault);
    cudaStream_t s = stream.get();
    DeviceArray<unsigned char> buf;
    buf.reserve(ar.bytes, s);
    CT_CUDA_CHECK(cudaMemcpyAsync(at<cticp_pose>(buf, o_gt), gt, sizeof(cticp_pose) * n, cudaMemcpyHostToDevice, s));
    PrepArgs p{};
    p.gt = at<cticp_pose>(buf, o_gt);
    p.n = (uint32_t) n;
    p.task = kPrepDistances;
    p.kind = kind;
    p.dist = at<double>(buf, o_dist);
    p.count = at<long long>(buf, o_count);
    k_prep<<<1, kPrepThreads, 0, s>>>(p);
    CT_CUDA_CHECK(cudaGetLastError());
    CT_CUDA_CHECK(cudaMemcpyAsync(out, p.dist, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
}

}  // namespace cticp
