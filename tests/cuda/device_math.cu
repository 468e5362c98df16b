// device_math.cu — test harness over the engine's own device math (tests/test_gpu_device_math.py).
//
// Includes the engine's headers and runs their routines unchanged, one extern "C" entry per routine, on B cases at once.
// Each entry copies its host arrays to the device, launches, copies the results back, frees everything and returns the
// cudaError_t of the sequence (0 = success). Every routine keeps the lane mapping it has in the engine: one thread per
// case for the scalar routines, one warp per case for the 12x12 solves and the Gauss-Newton step, and one half-warp per
// residual for ct_residual (lane hl computes tangent hl, lane 12 the value, as in lm_eval_device of icp_lm.cu).
//
// Built by ct_icp_b200/csrc/Makefile (target device_math) with the library's NVFLAGS: the contraction and optimisation
// flags are the library's, so the arithmetic is the arithmetic the engine runs. Test infrastructure, not part of the
// library.
#include <cuda_runtime.h>

#include <cstddef>

#include "gather_select.cuh"
#include "gn_step.cuh"
#include "lm_functor.cuh"
#include "small_solve.cuh"

using namespace cticp;

namespace {

// device copy of a host array, freed on scope exit
template <typename T>
struct Dev {
    T *p = nullptr;
    size_t n = 0;
    cudaError_t err = cudaSuccess;
    Dev(const T *host, size_t count) : n(count) {
        err = cudaMalloc(&p, sizeof(T) * (n ? n : 1));
        if (err == cudaSuccess && host) err = cudaMemcpy(p, host, sizeof(T) * n, cudaMemcpyHostToDevice);
        if (err == cudaSuccess && !host) err = cudaMemset(p, 0, sizeof(T) * (n ? n : 1));
    }
    ~Dev() {
        if (p) cudaFree(p);
    }
    Dev(const Dev &) = delete;
    Dev &operator=(const Dev &) = delete;
    cudaError_t to_host(T *host) const { return cudaMemcpy(host, p, sizeof(T) * n, cudaMemcpyDeviceToHost); }
};

int blocks_for(int threads, int per_block) { return (threads + per_block - 1) / per_block; }

// first error of a list of steps
cudaError_t first(std::initializer_list<cudaError_t> errs) {
    for (cudaError_t e : errs)
        if (e != cudaSuccess) return e;
    return cudaSuccess;
}
cudaError_t finish() {
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    return cudaDeviceSynchronize();
}

// ---- 3x3 symmetric eigen-decomposition ---------------------------------------------------------------------------------
// in: a00 a01 a02 a11 a12 a22. out (12): sv0 sv1 sv2, normal (3), line (3, full only), 3 unused
__global__ void k_sym_eig3(int full, int B, const double *a, double *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const double *c = a + 6 * i;
    double *o = out + 12 * i;
    if (full) {
        const Eig3Full e = sym_eig3_full(c[0], c[1], c[2], c[3], c[4], c[5]);
        o[0] = e.sv0; o[1] = e.sv1; o[2] = e.sv2;
        o[3] = e.normal.x; o[4] = e.normal.y; o[5] = e.normal.z;
        o[6] = e.line.x; o[7] = e.line.y; o[8] = e.line.z;
    } else {
        const Eig3 e = sym_eig3_fast(c[0], c[1], c[2], c[3], c[4], c[5]);
        o[0] = e.sv0; o[1] = e.sv1; o[2] = e.sv2;
        o[3] = e.normal.x; o[4] = e.normal.y; o[5] = e.normal.z;
        o[6] = o[7] = o[8] = 0.0;
    }
    o[9] = o[10] = o[11] = 0.0;
}

// ---- neighbourhood description from moments --------------------------------------------------------------------------
// rel: 32 x 3 offsets of the neighbours from the query per case (n[i] used). The moments are accumulated in neighbour
// order, the way one lane of warp_gather_sums accumulates its candidates (a[0..8]).
// out (16): describe_from_sums: normal (3), a2D, 12 unused; describe_full_from_sums: cov (6), normal (3), line (3),
// planarity, linearity, 2 unused
__global__ void k_describe(int full, int B, const int *n, const double *rel, double *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    double a[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    const double *r = rel + 96 * i;
    const int cnt = n[i] < 32 ? n[i] : 32;
    for (int k = 0; k < cnt; ++k) {
        const double x = r[3 * k], y = r[3 * k + 1], z = r[3 * k + 2];
        a[0] += x; a[1] += y; a[2] += z;
        a[3] += x * x; a[4] += x * y; a[5] += x * z;
        a[6] += y * y; a[7] += y * z; a[8] += z * z;
    }
    NeighborSums s;
    s.n = cnt;
    s.sx = a[0]; s.sy = a[1]; s.sz = a[2];
    s.sxx = a[3]; s.sxy = a[4]; s.sxz = a[5];
    s.syy = a[6]; s.syz = a[7]; s.szz = a[8];
    s.fx = s.fy = s.fz = s.fd2 = 0.0;
    double *o = out + 16 * i;
    for (int k = 0; k < 16; ++k) o[k] = 0.0;
    if (full) {
        const NeighborhoodDescFull d = describe_full_from_sums(s);
        for (int k = 0; k < 6; ++k) o[k] = d.cov[k];
        o[6] = d.normal.x; o[7] = d.normal.y; o[8] = d.normal.z;
        o[9] = d.line.x; o[10] = d.line.y; o[11] = d.line.z;
        o[12] = d.planarity; o[13] = d.linearity;
    } else {
        const NeighborhoodDesc d = describe_from_sums(s);
        o[0] = d.normal.x; o[1] = d.normal.y; o[2] = d.normal.z;
        o[3] = d.a2D;
    }
}

// ---- 12x12 solves: one warp per system -------------------------------------------------------------------------------
constexpr int kWarpsPerBlock = 4;

__global__ void k_ldlt(int compact, int B, const double *A, const double *b, double *x) {
    __shared__ SolveScratch sh[kWarpsPerBlock];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * kWarpsPerBlock + w;
    if (i >= B) return;   // whole warps leave together
    SolveScratch &S = sh[w];
    for (int e = lane; e < 144; e += 32) S.A[e / 12][e % 12] = A[144 * i + e];
    if (lane < 12) S.b[lane] = b[12 * i + lane];
    __syncwarp();
    if (compact) warp_ldlt_solve12_compact(S, lane);
    else warp_ldlt_solve12(S, lane);
    if (lane < 12) x[12 * i + lane] = S.x[lane];
}

// ---- Gauss-Newton step: one warp per case ----------------------------------------------------------------------------
// in (24): qb (4) tb (3) qe (4) te (3) prev_tb (3) prev_te (3) has_motion_model beta_location beta_cv, 1 unused
// out (40): qb tb qe te after the step (14), step x (12), x_norm, failed, done, iter, n_used, slerp theta, inv_sin,
// linear, negate, 4 unused.  sys (157): A (144), b (12), n_used — written by the solve itself (its debug tap).
constexpr int kGnIn = 24, kGnOut = 40, kGnSys = 157;

__global__ void k_gn_solve(int mode, int B, const double *acc, const double *in, double threshold_norm, double *out,
                           double *sys) {
    __shared__ SolveScratch sh[kWarpsPerBlock];
    __shared__ IcpState st_sh[kWarpsPerBlock];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * kWarpsPerBlock + w;
    if (i >= B) return;
    SolveScratch &S = sh[w];
    IcpState &st = st_sh[w];
    const double *p = in + kGnIn * i;
    if (lane == 0) {
        IcpState z = {};
        for (int d = 0; d < 4; ++d) { z.qb[d] = p[d]; z.qe[d] = p[7 + d]; }
        for (int d = 0; d < 3; ++d) {
            z.tb[d] = p[4 + d]; z.te[d] = p[11 + d];
            z.prev_tb[d] = p[14 + d]; z.prev_te[d] = p[17 + d];
        }
        z.has_motion_model = p[20] != 0.0;
        z.beta_location = p[21];
        z.beta_cv = p[22];
        st = z;
    }
    if (lane < 12) S.x[lane] = 0.0;
    __syncwarp();
    GnParams P = {};
    P.threshold_norm = threshold_norm;
    warp_gn_solve(acc + kAcc * i, S, &st, P, mode, sys + kGnSys * i, lane);
    __syncwarp();
    if (lane == 0) {
        double *o = out + kGnOut * i;
        for (int d = 0; d < 4; ++d) { o[d] = st.qb[d]; o[7 + d] = st.qe[d]; }
        for (int d = 0; d < 3; ++d) { o[4 + d] = st.tb[d]; o[11 + d] = st.te[d]; }
        for (int d = 0; d < 12; ++d) o[14 + d] = S.x[d];
        o[26] = st.x_norm;
        o[27] = st.failed; o[28] = st.done; o[29] = st.iter; o[30] = st.n_used;
        o[31] = st.slerp_theta; o[32] = st.slerp_inv_sin; o[33] = st.slerp_linear; o[34] = st.slerp_negate;
        for (int d = 35; d < kGnOut; ++d) o[d] = 0.0;
    }
}

// ---- CT functor: one half-warp per residual --------------------------------------------------------------------------
// blk (17): ref (3) normal (3) weight alpha raw (3) info (6); kind: kResPlane / kResLine / kResDistribution [| kResSimple]
// x (14): qb (4) qe (4) tb (3) te (3). out (13): 12 partials (tangent order), value
constexpr int kBlk = 17;

__device__ ResidualBlock make_block(const double *b, int kind) {
    ResidualBlock rb;
    for (int d = 0; d < 3; ++d) { rb.ref[d] = b[d]; rb.normal[d] = b[3 + d]; rb.raw[d] = b[8 + d]; }
    rb.weight = b[6];
    rb.alpha = b[7];
    for (int d = 0; d < 6; ++d) rb.info[d] = b[11 + d];
    rb.valid = 1;
    rb.kind = kind;
    return rb;
}

__global__ void k_ct_residual(int robust, int B, const double *blk, const int *kind, const double *x, double *out) {
    const int lane = threadIdx.x & 31, hl = lane & 15;
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 4;
    if (i >= B) return;   // half-warps leave together
    const ResidualBlock rb = make_block(blk + kBlk * i, kind[i]);
    const double *p = x + 14 * i;
    double qb[4], qe[4], tb[3], te[3];
    for (int d = 0; d < 4; ++d) { qb[d] = p[d]; qe[d] = p[4 + d]; }
    for (int d = 0; d < 3; ++d) { tb[d] = p[8 + d]; te[d] = p[11 + d]; }
    const Dual r = robust ? ct_residual<true>(rb, qb, qe, tb, te, hl) : ct_residual<false>(rb, qb, qe, tb, te, hl);
    if (hl < 12) out[13 * i + hl] = r.d;
    if (hl == 12) out[13 * i + 12] = r.a;
}

// value of dq_dot(dq_normalized(Qb), dq_normalized(Qe)) as ct_residual forms it before the slerp branch
__global__ void k_dq_dot(int B, const double *x, double *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const double *p = x + 14 * i;
    const DQuat Qb{mkd(p[0]), mkd(p[1]), mkd(p[2]), mkd(p[3])};
    const DQuat Qe{mkd(p[4]), mkd(p[5]), mkd(p[6]), mkd(p[7])};
    out[i] = dq_dot(dq_normalized(Qb), dq_normalized(Qe)).a;
}

// ---- scalar routines ---------------------------------------------------------------------------------------------------
__global__ void k_quat_plus(int B, const double *q, const double *d, double *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const Q4 r = quat_plus(Q4{q[4 * i], q[4 * i + 1], q[4 * i + 2], q[4 * i + 3]}, d[3 * i], d[3 * i + 1], d[3 * i + 2]);
    out[4 * i] = r.x; out[4 * i + 1] = r.y; out[4 * i + 2] = r.z; out[4 * i + 3] = r.w;
}

// loss (3): type, ls_sigma, ls_tolerant_min_threshold (make_loss as the LM setup calls it); out (3): rho
__global__ void k_loss(int B, const double *loss, const double *s, double *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const LossParams L = make_loss((int) loss[3 * i], loss[3 * i + 1], loss[3 * i + 2]);
    loss_evaluate(L, s[i], out + 3 * i);
}

// out (2): residual scale, jacobian scale
__global__ void k_corrector(int B, const double *s, const double *rho, double *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    corrector_1d(s[i], rho + 3 * i, out[2 * i], out[2 * i + 1]);
}

// in (18): qb (4) tb (3) qe (4) te (3) raw (3) alpha; out (12): ct_transform_c (3), qslerp_c (4) unnormalised, slerp
// constants theta, inv_sin, linear, negate, 1 unused
__global__ void k_ct_transform(int B, const double *in, double *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const double *p = in + 18 * i;
    const Q4 qb{p[0], p[1], p[2], p[3]}, qe{p[7], p[8], p[9], p[10]};
    const V3 tb{p[4], p[5], p[6]}, te{p[11], p[12], p[13]}, raw{p[14], p[15], p[16]};
    const SlerpConsts c = slerp_consts(qb, qe);
    const V3 w = ct_transform_c(qb, tb, qe, te, p[17], raw, c);
    const Q4 q = qslerp_c(qb, qe, p[17], c);
    double *o = out + 12 * i;
    o[0] = w.x; o[1] = w.y; o[2] = w.z;
    o[3] = q.x; o[4] = q.y; o[5] = q.z; o[6] = q.w;
    o[7] = c.theta; o[8] = c.inv_sin; o[9] = c.linear; o[10] = c.negate; o[11] = 0.0;
}

// R (9, row-major) -> q (4); q -> R
__global__ void k_qfromR(int B, const double *R, double *q) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    M3 m;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) m.m[r][c] = R[9 * i + 3 * r + c];
    const Q4 o = qfromR(m);
    q[4 * i] = o.x; q[4 * i + 1] = o.y; q[4 * i + 2] = o.z; q[4 * i + 3] = o.w;
}
__global__ void k_qtoR(int B, const double *q, double *R) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const M3 m = qtoR(Q4{q[4 * i], q[4 * i + 1], q[4 * i + 2], q[4 * i + 3]});
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) R[9 * i + 3 * r + c] = m.m[r][c];
}

// voxel_coord_rcp(p, res, 1 / res) with the reciprocal formed on the device like the map level does
__global__ void k_voxel_coord(int B, const double *p, double res, int *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    out[i] = voxel_coord_rcp(p[i], res, 1.0 / res);
}

}  // namespace

extern "C" {

int dm_sym_eig3(int full, int B, const double *a6, double *out12) {
    Dev<double> a(a6, 6 * (size_t) B), o(nullptr, 12 * (size_t) B);
    if (cudaError_t e = first({a.err, o.err})) return e;
    k_sym_eig3<<<blocks_for(B, 128), 128>>>(full, B, a.p, o.p);
    if (cudaError_t e = finish()) return e;
    return o.to_host(out12);
}

int dm_describe(int full, int B, const int *n, const double *rel96, double *out16) {
    Dev<int> dn(n, B);
    Dev<double> r(rel96, 96 * (size_t) B), o(nullptr, 16 * (size_t) B);
    if (cudaError_t e = first({dn.err, r.err, o.err})) return e;
    k_describe<<<blocks_for(B, 128), 128>>>(full, B, dn.p, r.p, o.p);
    if (cudaError_t e = finish()) return e;
    return o.to_host(out16);
}

int dm_ldlt_solve12(int compact, int B, const double *A144, const double *b12, double *x12) {
    Dev<double> A(A144, 144 * (size_t) B), b(b12, 12 * (size_t) B), x(nullptr, 12 * (size_t) B);
    if (cudaError_t e = first({A.err, b.err, x.err})) return e;
    k_ldlt<<<blocks_for(B, kWarpsPerBlock), 32 * kWarpsPerBlock>>>(compact, B, A.p, b.p, x.p);
    if (cudaError_t e = finish()) return e;
    return x.to_host(x12);
}

int dm_gn_solve(int mode, int B, const double *acc96, const double *in24, double threshold_norm, double *out40,
                double *sys157) {
    Dev<double> acc(acc96, (size_t) kAcc * B), in(in24, (size_t) kGnIn * B), out(nullptr, (size_t) kGnOut * B),
        sys(nullptr, (size_t) kGnSys * B);
    if (cudaError_t e = first({acc.err, in.err, out.err, sys.err})) return e;
    k_gn_solve<<<blocks_for(B, kWarpsPerBlock), 32 * kWarpsPerBlock>>>(mode, B, acc.p, in.p, threshold_norm, out.p, sys.p);
    if (cudaError_t e = finish()) return e;
    if (cudaError_t e = out.to_host(out40)) return e;
    return sys.to_host(sys157);
}

int dm_ct_residual(int robust, int B, const double *blk17, const int *kind, const double *x14, double *out13) {
    Dev<double> blk(blk17, (size_t) kBlk * B), x(x14, 14 * (size_t) B), o(nullptr, 13 * (size_t) B);
    Dev<int> k(kind, B);
    if (cudaError_t e = first({blk.err, x.err, o.err, k.err})) return e;
    k_ct_residual<<<blocks_for(16 * B, 128), 128>>>(robust, B, blk.p, k.p, x.p, o.p);
    if (cudaError_t e = finish()) return e;
    return o.to_host(out13);
}

int dm_dq_dot(int B, const double *x14, double *out) {
    Dev<double> x(x14, 14 * (size_t) B), o(nullptr, B);
    if (cudaError_t e = first({x.err, o.err})) return e;
    k_dq_dot<<<blocks_for(B, 128), 128>>>(B, x.p, o.p);
    if (cudaError_t e = finish()) return e;
    return o.to_host(out);
}

int dm_quat_plus(int B, const double *q4, const double *d3, double *out4) {
    Dev<double> q(q4, 4 * (size_t) B), d(d3, 3 * (size_t) B), o(nullptr, 4 * (size_t) B);
    if (cudaError_t e = first({q.err, d.err, o.err})) return e;
    k_quat_plus<<<blocks_for(B, 128), 128>>>(B, q.p, d.p, o.p);
    if (cudaError_t e = finish()) return e;
    return o.to_host(out4);
}

int dm_loss_evaluate(int B, const double *loss3, const double *s, double *rho3) {
    Dev<double> l(loss3, 3 * (size_t) B), ds(s, B), o(nullptr, 3 * (size_t) B);
    if (cudaError_t e = first({l.err, ds.err, o.err})) return e;
    k_loss<<<blocks_for(B, 128), 128>>>(B, l.p, ds.p, o.p);
    if (cudaError_t e = finish()) return e;
    return o.to_host(rho3);
}

int dm_corrector(int B, const double *s, const double *rho3, double *out2) {
    Dev<double> ds(s, B), r(rho3, 3 * (size_t) B), o(nullptr, 2 * (size_t) B);
    if (cudaError_t e = first({ds.err, r.err, o.err})) return e;
    k_corrector<<<blocks_for(B, 128), 128>>>(B, ds.p, r.p, o.p);
    if (cudaError_t e = finish()) return e;
    return o.to_host(out2);
}

int dm_ct_transform(int B, const double *in18, double *out12) {
    Dev<double> in(in18, 18 * (size_t) B), o(nullptr, 12 * (size_t) B);
    if (cudaError_t e = first({in.err, o.err})) return e;
    k_ct_transform<<<blocks_for(B, 128), 128>>>(B, in.p, o.p);
    if (cudaError_t e = finish()) return e;
    return o.to_host(out12);
}

int dm_qfromR(int B, const double *R9, double *q4) {
    Dev<double> R(R9, 9 * (size_t) B), q(nullptr, 4 * (size_t) B);
    if (cudaError_t e = first({R.err, q.err})) return e;
    k_qfromR<<<blocks_for(B, 128), 128>>>(B, R.p, q.p);
    if (cudaError_t e = finish()) return e;
    return q.to_host(q4);
}

int dm_qtoR(int B, const double *q4, double *R9) {
    Dev<double> q(q4, 4 * (size_t) B), R(nullptr, 9 * (size_t) B);
    if (cudaError_t e = first({q.err, R.err})) return e;
    k_qtoR<<<blocks_for(B, 128), 128>>>(B, q.p, R.p);
    if (cudaError_t e = finish()) return e;
    return R.to_host(R9);
}

int dm_voxel_coord_rcp(int B, const double *p, double res, int *out) {
    Dev<double> dp(p, B);
    Dev<int> o(nullptr, B);
    if (cudaError_t e = first({dp.err, o.err})) return e;
    k_voxel_coord<<<blocks_for(B, 128), 128>>>(B, dp.p, res, o.p);
    if (cudaError_t e = finish()) return e;
    return o.to_host(out);
}

}  // extern "C"
