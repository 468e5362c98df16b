// icp_gn.cu — Gauss-Newton CT-ICP iteration as two kernels per iteration:
//   k_gn_gather : one warp per keypoint — world point from the continuous-time pose pair, 27-voxel stencil gather,
//                 kNN, covariance + eigen, point-to-plane residual and 12-vector Jacobian row, accumulation of
//                 JTJ (78 unique entries) / JTr (12) in registers, block reduction in shared memory.
//   k_gn_solve  : one block — deterministic reduction of the per-block partials, 1/n normalisation, motion-model
//                 regularisers, pivoted LDL^T solve of the 12x12 system, Euler-ZYX pose update, stop test.
// Reference: DoRegisterGaussNewton, src/ct_icp/ct_icp.cpp:709-996 (serial per-keypoint loop :753-857).
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include <cooperative_groups.h>

#include "gather_select.cuh"
#include "icp.h"
#include "frame_policy.h"
#include "peer_exchange.cuh"
#include "small_solve.cuh"

namespace cticp {
namespace cg = cooperative_groups;

#define CT_CUDA_CHECK(expr)                                                                              \
    do {                                                                                                 \
        cudaError_t _e = (expr);                                                                         \
        if (_e != cudaSuccess)                                                                           \
            throw CudaError(std::string(#expr) + ": " + cudaGetErrorString(_e) + " @" + __FILE__ + ":" + \
                            std::to_string(__LINE__));                                                   \
    } while (0)

// Warps per CTA of the gather kernels (one keypoint per warp at a time). Fewer, fatter CTAs make the grid-wide
// barriers and the reduction of the per-CTA partial sums cheaper, and more warps share one SM's instruction cache: on
// config 2 (K ~ 1.2k) the GN loop per frame got faster from 4 to 8 to 16 warps (CTICP_GATHER_WARPS selects it)
// (16 warps x 128 registers = the whole register file: one CTA per SM, ~77 CTAs).
#ifndef CTICP_GATHER_WARPS
#define CTICP_GATHER_WARPS 16
#endif
constexpr int kGatherWarps = CTICP_GATHER_WARPS;



struct GatherLaunch {
    GatherConfig G;
    GnParams P;
};

__device__ __forceinline__ M3 euler_from_sincos(double sa, double ca, double sb, double cb, double sg, double cg) {
    M3 R;   // ct_icp.cpp:916-932
    R.m[0][0] = cg * cb; R.m[0][1] = -sg * ca + cg * sb * sa; R.m[0][2] = sg * sa + cg * sb * ca;
    R.m[1][0] = sg * cb; R.m[1][1] = cg * ca + sg * sb * sa;  R.m[1][2] = -cg * sa + sg * sb * ca;
    R.m[2][0] = -sb;     R.m[2][1] = cb * sa;                 R.m[2][2] = cb * ca;
    return R;
}

// One warp: accumulator (96 doubles in `acc`) → normal equations → GN step → pose update (ct_icp.cpp:860-980).
// mode 0: full step. mode 1: only emit the linear system into sys_out (debug tap).
__device__ __noinline__ void warp_gn_solve(const double *acc, SolveScratch &S, IcpState *st, const GnParams &P, int mode,
                              double *sys_out, int lane) {
    const int n_used = (int) (acc[kAccUsed] + 0.5);
    if (lane == 0) {
        st->n_used = n_used;
        st->n_keypoints = (int) (acc[kAccKeypoints] + 0.5);
        st->stat_keypoint_iters += (unsigned long long) (acc[kAccKeypoints] + 0.5);
        st->stat_stencil_points += (unsigned long long) (acc[kAccStencil] + 0.5);
        if (sys_out) sys_out[156] = (double) n_used;
    }
    if (n_used < 100) {   // ct_icp.cpp:860-871
        if (lane == 0) {
            st->failed = 1;
            st->done = 1;
        }
        return;
    }
    {
        const double inv = 1.0 / (double) n_used;   // :877-882
        for (int e = lane; e < 78; e += 32) {
            const int i = c_pair_i[e], j = c_pair_j[e];
            const double v = acc[e] * inv;
            S.A[i][j] = v;
            S.A[j][i] = v;
        }
        if (lane < 12) S.b[lane] = acc[78 + lane] * inv;
    }
    __syncwarp();
    if (st->has_motion_model && lane < 3) {   // :885-910
        const int d = lane;
        const double ac = st->beta_location, ae = st->beta_cv;
        const double diff_traj = st->tb[d] - st->te[d];   // the frame's own begin - end (sic, :892)
        S.A[3 + d][3 + d] += ac;
        S.b[3 + d] -= ac * diff_traj;
        const double diff_ego = st->te[d] - st->tb[d] - st->prev_te[d] + st->prev_tb[d];
        S.A[9 + d][9 + d] += ae;
        S.b[9 + d] -= ae * diff_ego;
    }
    __syncwarp();
    if (sys_out) {
        for (int e = lane; e < 144; e += 32) sys_out[e] = S.A[e / 12][e % 12];
        if (lane < 12) sys_out[144 + lane] = S.b[lane];
    }
    if (mode == 1) return;

    CT_STAMP(const long long t_ldlt = clock64();)
    warp_ldlt_solve12(S, lane);   // :914
    CT_STAMP(if (lane == 0) st->dbg_t[2] += (unsigned long long) (clock64() - t_ldlt);)
    CT_STAMP(const long long t_pose = clock64();)
    {
        // A rank-deficient system (all keypoints on one plane and no regulariser, …) gives a non-finite step where Eigen's
        // pivoted LDL^T would still return something bounded: report the failure instead of propagating NaN poses
        const bool finite = lane >= 12 || isfinite(S.x[lane]);
        if (!__all_sync(0xffffffffu, finite)) {
            if (lane == 0) {
                st->failed = 4;
                st->done = 1;
            }
            return;
        }
    }

    if (lane < 6) {   // angles x[0..2] (begin) and x[6..8] (end): sin / cos evaluated by six lanes at once
        const double ang = S.x[lane < 3 ? lane : lane + 3];
        // a GN step's angles are a fraction of a degree: polynomials (se3.cuh) instead of libm's argument reduction
        const bool small = fabs(ang) <= 0.5;
        S.sn[lane] = small ? sin_upto_half(ang) : sin(ang);
        S.cs[lane] = small ? cos_upto_half(ang) : cos(ang);
    }
    __syncwarp();
    if (lane < 2) {   // lane 0: begin pose, lane 1: end pose (:916-962)
        const int o = 3 * lane;
        const M3 R = euler_from_sincos(S.sn[o], S.cs[o], S.sn[o + 1], S.cs[o + 1], S.sn[o + 2], S.cs[o + 2]);
        double *qp = lane == 0 ? st->qb : st->qe;
        double *tp = lane == 0 ? st->tb : st->te;
        const Q4 q = qnormalized(qfromR(mmul(R, qtoR(Q4{qp[0], qp[1], qp[2], qp[3]}))));
        qp[0] = q.x; qp[1] = q.y; qp[2] = q.z; qp[3] = q.w;
        const int xo = lane == 0 ? 3 : 9;
        for (int d = 0; d < 3; ++d) tp[d] += S.x[xo + d];
    }
    __syncwarp();
    if (lane == 0) {
        double nrm = 0;
        for (int i = 0; i < 12; ++i) nrm += S.x[i] * S.x[i];
        nrm = sqrt(nrm);
        st->x_norm = nrm;
        st->iter += 1;
        if (nrm < P.threshold_norm) st->done = 1;   // :978
        const SlerpConsts sc = slerp_consts(Q4{st->qb[0], st->qb[1], st->qb[2], st->qb[3]},
                                            Q4{st->qe[0], st->qe[1], st->qe[2], st->qe[3]});
        st->slerp_theta = sc.theta;
        st->slerp_inv_sin = sc.inv_sin;
        st->slerp_linear = sc.linear;
        st->slerp_negate = sc.negate;
        CT_STAMP(st->dbg_t[3] += (unsigned long long) (clock64() - t_pose);)
    }
}

// ---- the gather half of an iteration: tiles of keypoints, grabbed by the warps of a CTA ---------------------------------
// A CTA owns a contiguous, balanced RANGE of the keypoints (static: keypoints c K / G .. (c + 1) K / G of G gather CTAs).
// Inside the CTA the warps grab TILES of W consecutive keypoints of that range from a shared-memory counter until the range
// is exhausted (one keypoint per grab while the range is no longer than two rounds of the CTA's warps, else ceil(range / warps), at
// most 16, when throughput counts). Per tile:
//   A  lane j < W : keypoint j's world position from the pose pair (slerp: two sin, one rsqrt) and its voxel (three
//                   fp64 divisions)                                                  [once per keypoint, not per lane]
//   B  all lanes  : for j = 0..W-1 the warp-cooperative gather + selection of gather_select.cuh; lane j keeps the moments
//   C  lane j < W : covariance → closed-form eigen → normal, a2D, residual, 12-vector Jacobian row → the CTA's row table
// and, when every row of the range is there, the CTA reduces the rows IN KEYPOINT ORDER into the 90 accumulators
// (gn_cta_reduce_rows): the result does not depend on which warp computed which row, so the work can be handed out
// dynamically — a warp whose keypoint has a sparse stencil takes the next one while a neighbour is still busy with a
// dense one — and the registration stays bit-reproducible. Per-warp clock64 stamps of the static tiles of
// two that came before showed a long tail of slow tiles, and every iteration waited for the slowest while half of the
// warps had no tile at all.
struct GnPose {
    Q4 qb, qe;
    V3 tb, te;
    SlerpConsts sc;
};
struct GnWarpAcc {
    double sum_sq = 0;               // (unused: Σ scalar² comes out of the CTA's row reduction, accumulator kAccSumSq)
    unsigned n_stencil = 0;          // per-lane partial counters
    int n_used = 0, n_kp = 0, n_valid = 0;
    CT_STAMP(long long dbg[4] = {0, 0, 0, 0};)   // cycles in phases A, B, C, D
};
constexpr int kDbgIters = 8, kDbgSlots = 6;

constexpr int kTileMax = 16;   // keypoints per warp tile (phases A / C cost 1/W per keypoint: 16 is deep in the flat part)
constexpr int kRowCap = 256;   // rows of a CTA's range held in shared memory at a time (longer ranges go in chunks)
constexpr int kRowParts = 5;   // the row reduction splits the rows over 5 x 96 threads

// Per-warp shared memory of a tile: the gather's staging area and the moments of each keypoint of the tile (phase B hands
// them to phase C through here instead of through 27 registers that would stay live across the gather).
struct __align__(16) TileScratch {
    SelScratch sel;
    double sums[kTileMax][14];   // NeighborSums of keypoint j: n, stencil points, s*, f*
};
// Per-CTA row table of the current chunk of the CTA's range
struct __align__(16) CtaRows {
    double u[kRowCap][13];       // u[0..11], -scalar of keypoint (chunk base + r); valid iff used[r]
    unsigned char used[kRowCap];
    double red[kRowParts][kAcc];
    int next;                    // tile counter of the chunk
};

// keypoints per tile for a CTA range of `span` keypoints
__device__ __forceinline__ int gn_tile_width(int span) {
    // one keypoint per grab while the range is at most two rounds of the CTA's warps (the loop is bound by the slowest
    // keypoint there: balance counts); beyond that one tile per warp, as wide as it gets (throughput: the lane-per-keypoint
    // phases cost 1/W per keypoint — on the dense workload, K = 32k, tiles of 7 were slower than tiles of 14)
    if (span <= 2 * CTICP_GATHER_WARPS) return 1;
    const int W = (span + CTICP_GATHER_WARPS - 1) / CTICP_GATHER_WARPS;
    return W < kTileMax ? W : kTileMax;
}

// The tiles of the chunk [lo, hi) of this CTA's range (hi - lo <= kRowCap); R.next must be 0 and visible (barrier) on entry.
__device__ __forceinline__ void gn_gather_tiles(const GatherLaunch &cfg, const int *stencil,
                                                const float4 *__restrict__ keypoints, int lo, int hi, int W,
                                                const GnPose &pose, TileScratch &T, CtaRows &R, int lane,
                                                GnWarpAcc &A, void *bulk = nullptr, bool rigid = false) {
    const GatherConfig &G = cfg.G;
    const GnParams &P = cfg.P;
    if (hi <= lo) return;
    const int need = P.kmin > 5 ? P.kmin : 5;   // ct_icp.cpp:769 ; neighborhood.h:227
    const double inv_res = 1.0 / G.L.res;

    while (true) {
        int j0 = 0;
        if (lane == 0) j0 = atomicAdd(&R.next, W);
        j0 = __shfl_sync(0xffffffffu, j0, 0);
        const int t0 = lo + j0;
        if (t0 >= hi) break;
        const int wt = (hi - t0) < W ? (hi - t0) : W;
        CT_STAMP(const long long t_a = clock64();)
        // ---- A: world_kpts[i] = InterpolatePose(begin, end, t_i) * raw_i  (ct_icp.cpp:964-966, types.h:361-366)
        V3 p{0, 0, 0};
        int kx = 0, ky = 0, kz = 0;
        if (lane < wt) {
            const RawPoint kraw = load_raw(keypoints, P.kp_lo, t0 + lane);   // raw xyz (sensor frame) + alpha timestamp
            const V3 raw{kraw.x, kraw.y, kraw.z};
            p = rigid ? qrot(qnormalized(pose.qe), raw) + pose.te
                      : ct_transform_c(pose.qb, pose.tb, pose.qe, pose.te, kraw.alpha, raw, pose.sc);
            kx = voxel_coord_rcp(p.x, G.L.res, inv_res);
            ky = voxel_coord_rcp(p.y, G.L.res, inv_res);
            kz = voxel_coord_rcp(p.z, G.L.res, inv_res);
        }
        CT_STAMP(const long long t_b = clock64();)
        // ---- B
        for (int j = 0; j < wt; ++j) {
            const V3 q{__shfl_sync(0xffffffffu, p.x, j), __shfl_sync(0xffffffffu, p.y, j), __shfl_sync(0xffffffffu, p.z, j)};
            const int qx = __shfl_sync(0xffffffffu, kx, j), qy = __shfl_sync(0xffffffffu, ky, j),
                      qz = __shfl_sync(0xffffffffu, kz, j);
            NeighborSums s;
            unsigned spts = 0;
            warp_gather_sums<false>(G, P.bucket_scale, stencil, q, qx, qy, qz, need, lane, T.sel, s, spts, V3{0, 0, 0}, bulk);
            if (lane == 0) {
                double *o = T.sums[j];
                o[0] = __hiloint2double((int) spts, s.n);   // two integers in one slot: no int <-> double conversion
                if (s.n >= need) {
                    o[2] = s.sx; o[3] = s.sy; o[4] = s.sz;
                    o[5] = s.sxx; o[6] = s.sxy; o[7] = s.sxz; o[8] = s.syy; o[9] = s.syz; o[10] = s.szz;
                    o[11] = s.fx; o[12] = s.fy; o[13] = s.fz;
                }
            }
        }
        __syncwarp();
        CT_STAMP(const long long t_c = clock64();)
        // ---- C (ct_icp.cpp:769-850)
        if (lane < wt) {
            bool used = false;
            const double *o = T.sums[lane];
            NeighborSums mine;
            mine.n = __double2loint(o[0]);
            A.n_kp += 1;
            A.n_stencil += (unsigned) __double2hiint(o[0]);
            if (mine.n >= need) {
                A.n_valid += 1;
                mine.sx = o[2]; mine.sy = o[3]; mine.sz = o[4];
                mine.sxx = o[5]; mine.sxy = o[6]; mine.sxz = o[7]; mine.syy = o[8]; mine.syz = o[9]; mine.szz = o[10];
                mine.fx = o[11]; mine.fy = o[12]; mine.fz = o[13]; mine.fd2 = 0;
                const NeighborhoodDesc nd = describe_from_sums(mine);
                V3 normal = nd.normal;
                // orient towards the sensor position at frame begin (:782-784)
                if (dot(normal, pose.tb - p) < 0) normal = -1.0 * normal;
                const double weight = nd.a2D * nd.a2D;                       // :787-788
                // p - closest_point, closest_point = points[0] = farthest kept (:791)
                const V3 diff{-nd.far_rel.x, -nd.far_rel.y, -nd.far_rel.z};
                const double dist_to_plane = dot(normal, diff);
                if (fabs(dist_to_plane) < P.max_dist_to_plane) {              // :803
                    const V3 nw = weight * normal;
                    const double scalar = dot(nw, diff);
                    const RawPoint kraw = load_raw(keypoints, P.kp_lo, t0 + lane);
                    const V3 raw{kraw.x, kraw.y, kraw.z};
                    const V3 ob = qrot(pose.qb, raw), oe = qrot(pose.qe, raw);   // :813-816
                    const double a = kraw.alpha, am = 1.0 - a;
                    const V3 cb = cross(ob, nw), ce = cross(oe, nw);
                    double *u = R.u[j0 + lane];
                    u[0] = am * cb.x; u[1] = am * cb.y; u[2] = am * cb.z;
                    u[3] = am * nw.x; u[4] = am * nw.y; u[5] = am * nw.z;
                    u[6] = a * ce.x;  u[7] = a * ce.y;  u[8] = a * ce.z;
                    u[9] = a * nw.x;  u[10] = a * nw.y; u[11] = a * nw.z;
                    u[12] = -scalar;   // b -= u * scalar (:849)
                    used = true;
                    A.n_used += 1;
                }
            }
            R.used[j0 + lane] = used ? 1 : 0;
        }
        __syncwarp();   // the moments are consumed before the next tile rewrites them
        CT_STAMP(const long long t_e = clock64();
                 A.dbg[0] += t_b - t_a; A.dbg[1] += t_c - t_b; A.dbg[2] += t_e - t_c;)
    }
}

// A += u u^T, b -= u scalar over the rows [0, n) of the chunk, in keypoint order within each of kRowParts interleaved
// classes, the classes then in fixed order: deterministic whatever warp wrote a row. Thread t < kRowParts * kAcc handles
// accumulator t % kAcc (entries 0..89: pairs of [A upper | b]; 90: rows used; 91: Σ scalar²) of class t / kAcc. The sum
// of the chunk is ADDED to `carry` of the threads < kAcc. Called by all threads of the CTA; barriers inside.
__device__ __forceinline__ void gn_cta_reduce_rows(CtaRows &R, int n, double &carry) {
    const int t = threadIdx.x;
    const int a = t % kAcc, part = t / kAcc;
    __syncthreads();   // every row of the chunk is written
    if (part < kRowParts && a <= kAccSumSq) {
        const int pi = a < kAccUsed ? c_pair_i[a] : 12, pj = a < kAccUsed ? c_pair_j[a] : 12;
        double s = 0;
        if (a == kAccUsed) {
            int c = 0;
            for (int r = part; r < n; r += kRowParts) c += R.used[r];
            s = i32_to_f64(c);
        } else {
            for (int r = part; r < n; r += kRowParts)
                if (R.used[r]) s += R.u[r][pi] * R.u[r][pj];
        }
        R.red[part][a] = s;
    }
    __syncthreads();
    if (t < kAcc && a <= kAccSumSq) {
        double s = R.red[0][a];
#pragma unroll
        for (int q = 1; q < kRowParts; ++q) s += R.red[q][a];
        carry += s;
    }
}

// per-warp counters → the warp's row of `kAcc` doubles in shared memory (the accumulators come from gn_cta_reduce_rows)
__device__ __forceinline__ void gn_store_warp_row(double *row, const GnWarpAcc &A, int lane) {
    const unsigned n_stencil = __reduce_add_sync(0xffffffffu, A.n_stencil);
    const int n_kp = __reduce_add_sync(0xffffffffu, A.n_kp), n_valid = __reduce_add_sync(0xffffffffu, A.n_valid);
    if (lane == 0) {
        row[kAccStencil] = i32_to_f64((int) n_stencil);
        row[kAccKeypoints] = i32_to_f64(n_kp);
        row[kAccValidNb] = i32_to_f64(n_valid);
    }
}

// The gather half of an iteration for one CTA: its range [c_lo, c_hi) of the keypoints in chunks of kRowCap rows →
// this CTA's partial row (kAcc doubles) in global memory. `R.next` is reset here; all threads call.
// shared memory of the GN kernels (dynamic: the staging areas alone are 70 KB)
struct GnShared {
    TileScratch tile[kGatherWarps];
    CtaRows rows;
    GnPose pose;
    double acc[kGatherWarps][kAcc];
    int stencil[kMaxStencil];
    SolveScratch solve;
    IcpState dummy;
    IcpState state;   // persistent kernel, solver CTA: the registration state lives here; `st` (global) is its published copy
    FrameVerdict verdict;   // persistent kernel, solver CTA: the frame's tail decided at the end of the loop (frame_policy.h)
    int flag;
    int done;         // gather CTAs: the published `done` flag, fetched together with the pose (one memory round trip)
    unsigned long long mbar[kGatherWarps];   // -DCTICP_SEL_BULK: one mbarrier per warp for the bulk copies
};

// deterministic reduction of `rows` partial rows by one CTA: warp g sums the rows b = g (mod kGatherWarps), three
// columns per lane, all of a warp's loads in flight before the first add; then the per-warp sums in fixed order.
// Result in sh.acc[0][0..kAcc). Called by all threads.
__device__ __forceinline__ void gn_reduce_rows(GnShared &sh, const double *__restrict__ partials, int rows, int lane, int w) {
    constexpr int kInFlight = 10;
    double a0 = 0, a1 = 0, a2 = 0;
    for (int b0 = w; b0 < rows; b0 += kGatherWarps * kInFlight) {
        double v0[kInFlight], v1[kInFlight], v2[kInFlight];
#pragma unroll
        for (int u = 0; u < kInFlight; ++u) {
            const int b = b0 + u * kGatherWarps;
            v0[u] = v1[u] = v2[u] = 0.0;
            if (b < rows) {
                const double *row = partials + (size_t) b * kAcc;
                v0[u] = __ldcg(row + lane);
                v1[u] = __ldcg(row + lane + 32);
                v2[u] = __ldcg(row + lane + 64);
            }
        }
#pragma unroll
        for (int u = 0; u < kInFlight; ++u)
            if (b0 + u * kGatherWarps < rows) {
                a0 += v0[u];
                a1 += v1[u];
                a2 += v2[u];
            }
    }
    __syncthreads();
    sh.acc[w][lane] = a0;
    sh.acc[w][lane + 32] = a1;
    sh.acc[w][lane + 64] = a2;
    __syncthreads();
    double sum = 0;
    if (threadIdx.x < kAcc) {
#pragma unroll
        for (int ww = 0; ww < kGatherWarps; ++ww) sum += sh.acc[ww][threadIdx.x];
    }
    __syncthreads();
    if (threadIdx.x < kAcc) sh.acc[0][threadIdx.x] = sum;
    __syncthreads();
}

// The gather half of an iteration for one CTA: its range [c_lo, c_hi) of the keypoints, in chunks of kRowCap rows →
// the CTA's partial row (kAcc doubles) at `partial_out` (global). On entry sh.pose is valid and sh.rows.next == 0, both
// visible to the CTA (the thread that fetched the pose set them before a barrier). All threads call.
__device__ __forceinline__ void gn_cta_gather(const GatherLaunch &cfg, const int *stencil, const float4 *__restrict__ keypoints,
                                              int c_lo, int c_hi, GnShared &sh, int lane, int w, double *partial_out,
                                              GnWarpAcc &A, void *bulk, bool rigid) {
    const int W = gn_tile_width(c_hi - c_lo);
    double carry = 0;
    for (int base = c_lo;; base += kRowCap) {
        const int top = (c_hi - base) > kRowCap ? base + kRowCap : c_hi;
        gn_gather_tiles(cfg, stencil, keypoints, base, top, W, sh.pose, sh.tile[w], sh.rows, lane, A, bulk, rigid);
        gn_cta_reduce_rows(sh.rows, top > base ? top - base : 0, carry);
        if (top >= c_hi) break;
        if (threadIdx.x == 0) sh.rows.next = 0;
        __syncthreads();
    }
    gn_store_warp_row(sh.acc[w], A, lane);
    __syncthreads();
    if (threadIdx.x < kAcc) {
        const int t = threadIdx.x;
        double s = 0;
        if (t <= kAccSumSq) s = carry;
        else if (t == kAccStencil || t == kAccKeypoints || t == kAccValidNb) {
#pragma unroll
            for (int ww = 0; ww < kGatherWarps; ++ww) s += sh.acc[ww][t];
        }
        __stcg(partial_out + t, s);
    }
}

__device__ __forceinline__ GnPose load_pose(const IcpState *st) {
    GnPose p;
    p.qb = Q4{__ldcg(&st->qb[0]), __ldcg(&st->qb[1]), __ldcg(&st->qb[2]), __ldcg(&st->qb[3])};
    p.qe = Q4{__ldcg(&st->qe[0]), __ldcg(&st->qe[1]), __ldcg(&st->qe[2]), __ldcg(&st->qe[3])};
    p.tb = V3{__ldcg(&st->tb[0]), __ldcg(&st->tb[1]), __ldcg(&st->tb[2])};
    p.te = V3{__ldcg(&st->te[0]), __ldcg(&st->te[1]), __ldcg(&st->te[2])};
    p.sc = SlerpConsts{__ldcg(&st->slerp_theta), __ldcg(&st->slerp_inv_sin), __ldcg(&st->slerp_linear), __ldcg(&st->slerp_negate)};
    return p;
}

static_assert(sizeof(GnShared) <= 227 * 1024, "k_gn_persistent: dynamic shared memory of one CTA (sm_90: 227 KB)");
extern __shared__ __align__(16) unsigned char gn_smem_raw[];

// mode 0: gather + (last CTA) reduce + solve + pose update          [one launch per ICP iteration]
// mode 1: gather + (last CTA) reduce + emit linear system to sys_out [debug tap]
// mode 2: gather + (last CTA) reduce into acc_out                    [multi-GPU over NCCL: all-reduce then k_gn_solve_acc]
__global__ void __launch_bounds__(kGatherWarps * 32, 1)
k_gn_iterate(GatherLaunch cfg, const float4 *__restrict__ keypoints, const int *__restrict__ d_num_keypoints,
             IcpState *st, double *__restrict__ partials, unsigned int *ticket, int mode, double *acc_out,
             double *sys_out) {
    GnShared &sh = *reinterpret_cast<GnShared *>(gn_smem_raw);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const GnParams &P = cfg.P;
    const bool active = (mode == 1) || !st->done;

    GnWarpAcc A;
    void *bulk_ptr = nullptr;
#ifdef CTICP_SEL_BULK
    SelBulk bulk;
    sel_bulk_init(bulk, &sh.mbar[w], lane);
    bulk_ptr = &bulk;
#endif
    {
        const int *stencil = stencil_table_fill(sh.stencil, cfg.G.r);
        if (threadIdx.x == 0) {
            sh.pose = load_pose(st);
            sh.rows.next = 0;
        }
        __syncthreads();
        int c_lo = 0, c_hi = 0;   // inactive (the registration has converged): an empty range, a zero partial row
        if (active) {
            const int K = *d_num_keypoints;
            const int lo = (int) ((long long) K * P.shard_rank / P.shard_world);
            const int hi = (int) ((long long) K * (P.shard_rank + 1) / P.shard_world);
            c_lo = lo + (int) ((long long) (hi - lo) * blockIdx.x / gridDim.x);
            c_hi = lo + (int) ((long long) (hi - lo) * (blockIdx.x + 1) / gridDim.x);
        }
        gn_cta_gather(cfg, stencil, keypoints, c_lo, c_hi, sh, lane, w, partials + (size_t) blockIdx.x * kAcc, A, bulk_ptr,
                      active && P.rigid_first && __ldcg(&st->iter) == 0);
    }
    // ---- last CTA to finish reduces the partials (fixed order) and takes the Gauss-Newton step -----------------
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) sh.flag = (atomicAdd(ticket, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!sh.flag) return;
    __threadfence();
    if (threadIdx.x == 0) {
        *ticket = 0;
    }
    if (!active) return;
    gn_reduce_rows(sh, partials, (int) gridDim.x, lane, w);
    if (mode == 2 && threadIdx.x < kAcc) acc_out[threadIdx.x] = sh.acc[0][threadIdx.x];
    if (mode == 2 || w != 0) return;
    warp_gn_solve(sh.acc[0], sh.solve, st, P, mode, sys_out, lane);
}

// ---- synchronisation of the persistent loop: two flags instead of two grid-wide barriers per iteration ------------------
// The loop's dependencies are asymmetric: the solver CTA needs every gather CTA's partial row; a gather CTA needs the solver
// CTA's new pose — it never needs the OTHER gather CTAs. So a gather CTA only ARRIVES (fence + one atomic, no wait) and then
// polls the epoch word the solver CTA bumps after publishing the state, and the solver CTA polls the arrival counter. Per
// iteration that is one L2 round trip on each side instead of two cg::grid.sync() (each a full
// grid-wide round trip; tools/micro/coop_launch_cost.cu measures one) plus the separate fetch of the pose.
// The launch stays cooperative: the CTAs must be co-resident for the polls to make progress. Every poll is bounded: a
// protocol error ends the kernel with st->failed = 2 instead of hanging the device.
// Two sets of words alternate between launches; the solver CTA of a launch zeroes the set of the NEXT launch (nobody touches
// it meanwhile), so no memset sits between the sampler and this kernel.
#ifndef CTICP_GN_GRID_BARRIERS
#define CTICP_GN_FLAG_SYNC 1
#endif
struct LoopSync {
    unsigned int *arrive;   // += 1 by every gather CTA at the end of its gather
    unsigned int *epoch;    // = iterations published by the solver CTA
    unsigned int *next_arrive, *next_epoch;   // the other set
};
constexpr long long kLoopSyncTimeout = 4000000000LL;   // SM cycles (~2 s)
__device__ __forceinline__ bool loop_wait_at_least(const unsigned int *word, unsigned int want,
                                                   long long timeout = kLoopSyncTimeout) {
    const long long t0 = clock64();
    while (*reinterpret_cast<const volatile unsigned int *>(word) < want)
        if (clock64() - t0 > timeout) return false;
    __threadfence();
    return true;
}

// ---- persistent variant: the WHOLE Gauss-Newton loop in one cooperative launch --------------------------------
// CTA 0 is the solver CTA (deterministic reduction of the partials + 12x12 solve + pose update, by the same warp on
// the same SM every iteration, so its instructions stay in that SM's instruction cache: executed cold, the serial tail
// costs tens of microseconds per iteration, warm a few); CTAs 1..G gather. The two sides meet through the arrive / epoch
// words above (-DCTICP_GN_GRID_BARRIERS: two grid-wide barriers per iteration, the round's earlier form). While the gather
// CTAs work on iteration 0, the solver warp runs the solve once on a dummy system to pull its code into the instruction
// cache. With `tail.enabled` the solver CTA also decides the frame's tail after the loop (frame_policy.h).
//
// kPeers (multi-GPU, keypoints sharded): between its reduction and its solve the solver CTA exchanges the accumulator
// with the other ranks' solver CTAs through NVLink peer memory (peer_exchange.cuh) — the all-reduce of SURVEY §8e
// happens INSIDE the loop, so the sharded loop is still one launch and costs one NVLink round trip per iteration.
template <bool kPeers>
__global__ void __launch_bounds__(kGatherWarps * 32, 1)
k_gn_persistent(GatherLaunch cfg, const float4 *__restrict__ keypoints, const int *__restrict__ d_num_keypoints,
                IcpState *st, double *__restrict__ partials, int num_iters, PeerLinks links, LoopSync sync,
                FrameTailArgs tail) {
#ifndef CTICP_GN_FLAG_SYNC
    cg::grid_group grid = cg::this_grid();
#endif
    GnShared &sh = *reinterpret_cast<GnShared *>(gn_smem_raw);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const GnParams &P = cfg.P;
    const bool solver_cta = blockIdx.x == 0;
#ifdef CTICP_GN_FLAG_SYNC
    if (solver_cta && threadIdx.x == 0) {   // the next launch's words (idle during this launch)
        *sync.next_arrive = 0u;
        *sync.next_epoch = 0u;
    }
#endif
    unsigned int peer_seq = 0;   // sequence number of the last exchange (solver CTA only)
    if (kPeers && solver_cta) peer_seq = *links.seq;
    const int gather_ctas = gridDim.x - 1;
    const int *stencil = stencil_table_fill(sh.stencil, cfg.G.r);
    __syncthreads();

    if (solver_cta) {   // working copy of the state in shared memory: the serial tail never waits for global memory
        const int *src = reinterpret_cast<const int *>(st);
        int *dst = reinterpret_cast<int *>(&sh.state);
        for (int i = threadIdx.x; i < (int) (sizeof(IcpState) / sizeof(int)); i += blockDim.x) dst[i] = src[i];
        __syncthreads();
    }
    CT_STAMP(if (solver_cta && threadIdx.x < 4) sh.state.dbg_t[threadIdx.x] = 0; __syncthreads();)
    if (solver_cta && w == 0 && !(P.debug_flags & 4)) {
        // instruction-cache warm-up of the serial tail on a dummy well-posed system (results discarded)
        for (int i = lane; i < kAcc; i += 32) sh.acc[1][i] = 0.0;
        __syncwarp();
        for (int e = lane; e < 78; e += 32)
            if (c_pair_i[e] == c_pair_j[e]) sh.acc[1][e] = 200.0 * (1.0 + c_pair_i[e]);
        if (lane < 12) sh.acc[1][78 + lane] = 1e-3 * (lane + 1);
        if (lane == 0) {
            sh.acc[1][kAccUsed] = 200.0;
            sh.dummy = sh.state;
        }
        __syncwarp();
        warp_gn_solve(sh.acc[1], sh.solve, &sh.dummy, P, 0, nullptr, lane);
        __syncwarp();
    }

    void *bulk_ptr = nullptr;
#ifdef CTICP_SEL_BULK
    SelBulk bulk;
    sel_bulk_init(bulk, &sh.mbar[w], lane);
    bulk_ptr = &bulk;
#endif
    long long t_loop = 0, t_solve = 0;
    if (solver_cta && threadIdx.x == 0) t_loop = clock64();
    // this rank's keypoint range and the tile width: constant over the iterations (integer divisions)
    const int K = *d_num_keypoints;
    int kp_lo = 0, kp_hi = K;
    if (P.shard_world > 1) {
        kp_lo = (int) ((long long) K * P.shard_rank / P.shard_world);
        kp_hi = (int) ((long long) K * (P.shard_rank + 1) / P.shard_world);
    }
    // this CTA's balanced share of the range
    int c_lo = 0, c_hi = 0;
    if (!solver_cta) {
        c_lo = kp_lo + (int) ((long long) (kp_hi - kp_lo) * (blockIdx.x - 1) / gather_ctas);
        c_hi = kp_lo + (int) ((long long) (kp_hi - kp_lo) * blockIdx.x / gather_ctas);
    }
    for (int it = 0; it < num_iters; ++it) {
        // `done` is uniform over the grid: published before the previous grid barrier (the solver CTA reads its own copy)
        if (solver_cta) {
            if (sh.state.done) break;
        } else {
            GnWarpAcc A;
            CT_STAMP(const long long t_it = clock64();)
            if (threadIdx.x == 0) {   // phases A / C read the pose from shared memory: 34 registers less to keep live
#ifdef CTICP_GN_FLAG_SYNC
                // the state of iteration `it` is published (it == 0: uploaded by the host before the launch)
                // (sharded: the solver CTA may itself be waiting for a late peer rank, up to PeerLinks::timeout_cycles)
                const bool ok = it == 0 || loop_wait_at_least(sync.epoch, (unsigned int) it,
                                                              kLoopSyncTimeout + (kPeers ? links.timeout_cycles : 0LL));
#else
                const bool ok = true;
#endif
                const int done = __ldcg(&st->done);   // issued with the pose loads: one round trip, not two
                sh.pose = load_pose(st);
                sh.done = ok ? done : 1;
                sh.rows.next = 0;
            }
            __syncthreads();
            if (sh.done) break;
            CT_STAMP(const long long t_g0 = clock64();)
            // (CTICP_DEBUG_FLAGS & 2, timing only: an empty range — the barriers and the reduction without the gather work)
            const bool skip = (P.debug_flags & 2) != 0;
            gn_cta_gather(cfg, stencil, keypoints, skip ? 0 : c_lo, skip ? 0 : c_hi, sh, lane, w,
                          partials + (size_t) (blockIdx.x - 1) * kAcc, A, bulk_ptr, P.rigid_first && it == 0);
            CT_STAMP(const long long t_g = clock64();)
#ifdef CTICP_GN_FLAG_SYNC
            __threadfence();   // (the writers of the partial row)
            __syncthreads();
            if (threadIdx.x == 0) atomicAdd(sync.arrive, 1u);
#endif
            CT_STAMP(if (P.dbg_warp && lane == 0 && it < kDbgIters) {
                unsigned long long *o = P.dbg_warp + ((size_t) it * (gather_ctas * kGatherWarps) + (w * gather_ctas + (blockIdx.x - 1))) * kDbgSlots;
                o[0] = (unsigned long long) A.dbg[0]; o[1] = (unsigned long long) A.dbg[1];
                o[2] = (unsigned long long) A.dbg[2];
                o[3] = (unsigned long long) (t_g0 - t_it);         // pose fetch + barrier
                o[4] = (unsigned long long) (t_g - t_it);          // pose fetch + tiles + CTA row reduction
                o[5] = 0;
            })
#ifdef CTICP_GN_FLAG_SYNC
            if (it == num_iters - 1) break;   // nothing left to wait for: the solver CTA finishes the registration alone
#endif
        }
        CT_STAMP(const long long t_bar = clock64();)
#ifdef CTICP_GN_FLAG_SYNC
        if (solver_cta) {
            if (threadIdx.x == 0) sh.flag = loop_wait_at_least(sync.arrive, (unsigned int) (gather_ctas * (it + 1))) ? 1 : 0;
            __syncthreads();
            if (!sh.flag) {   // a gather CTA never arrived: give up (the host raises "Error During Optimization")
                if (threadIdx.x == 0) {
                    sh.state.failed = 2;
                    sh.state.done = 1;
                    st->failed = 2;
                    st->done = 1;
                    __threadfence();
                    atomicExch(sync.epoch, 0x7fffffffu);
                }
                break;
            }
        }
#else
        grid.sync();
#endif
        CT_STAMP(if (!solver_cta && P.dbg_warp && lane == 0 && w == 0 && it < kDbgIters) {
            // (slot 5 of this CTA's first warp is overwritten with the wait at the barrier that follows the gather)
            unsigned long long *o = P.dbg_warp + ((size_t) it * (gather_ctas * kGatherWarps) + (blockIdx.x - 1)) * kDbgSlots;
            o[5] = (unsigned long long) (clock64() - t_bar);
        })
        if (solver_cta) {
            const long long t_begin = threadIdx.x == 0 ? clock64() : 0;
            gn_reduce_rows(sh, partials, gather_ctas, lane, w);
            // -DCTICP_DEBUG_TIMERS: SM cycles summed over the iterations — dbg_t[0] reduction of the partial rows,
            // [1] everything from there to the published state, [2] the 12x12 solve, [3] the pose update
            CT_STAMP(if (threadIdx.x == 0) sh.state.dbg_t[0] += (unsigned long long) (clock64() - t_begin);)
            CT_STAMP(const long long t_rest = clock64();)
            bool peers_ok = true;
            if (kPeers) {
                // Σ over ranks, in rank order (bit-identical on every rank); the staging areas are unused by the solver
                // CTA and serve as scratch
                static_assert(sizeof(TileScratch) * kGatherWarps >= sizeof(unsigned int) * kMaxPeers * kPeerWords, "scratch");
                peers_ok = peer_allreduce(links, ++peer_seq, sh.acc[0], reinterpret_cast<unsigned int *>(&sh.tile[0]), &sh.flag);
            }
            if (w == 0) {
                IcpState *ws = &sh.state;
                if (!peers_ok) {
                    if (lane == 0) {   // a peer never answered: give up instead of hanging the device
                        ws->failed = 3;
                        ws->done = 1;
                    }
                } else if (P.debug_flags & 1) {
                    if (lane == 0) ws->iter += 1;
                } else
                    warp_gn_solve(sh.acc[0], sh.solve, ws, P, 0, nullptr, lane);
                __syncwarp();
                if (lane == 0) {
                    t_solve += clock64() - t_begin;
                    ws->cycles_total = (unsigned long long) (clock64() - t_loop);
                    ws->cycles_solve = (unsigned long long) t_solve;
                }
                __syncwarp();
                // publish: the gather CTAs read the pose pair / done flag of the next iteration from global memory
                const int *src = reinterpret_cast<const int *>(ws);
                int *dst = reinterpret_cast<int *>(st);
                for (int i = lane; i < (int) (sizeof(IcpState) / sizeof(int)); i += 32) __stcg(dst + i, src[i]);
                CT_STAMP(if (lane == 0) {
                    ws->dbg_t[1] += (unsigned long long) (clock64() - t_rest);
                    __stcg(&st->dbg_t[1], ws->dbg_t[1]);
                })
#ifdef CTICP_GN_FLAG_SYNC
                __threadfence();   // (the lanes that wrote the state)
                __syncwarp();
                if (lane == 0) atomicExch(sync.epoch, (unsigned int) (it + 1));
#endif
            }
#ifdef CTICP_GN_FLAG_SYNC
            __syncthreads();   // warp 0 is done with sh.acc / sh.state before the next iteration's reduction
#else
            __threadfence();
#endif
        }
#ifndef CTICP_GN_FLAG_SYNC
        grid.sync();
#endif
    }
    if (kPeers && solver_cta && threadIdx.x == 0) *links.seq = peer_seq;
    // ---- the tail of the registration (frame_policy.h): AssessRegistration + the insertion policy on the final state, the
    // verdict to HBM (the speculative map update launched behind this kernel reads it) and to mapped pinned host memory
    if (solver_cta && tail.enabled) {
        __syncthreads();   // sh.state is final
        if (w == 0) {
            const int *src = reinterpret_cast<const int *>(&sh.state);
            int *dst = reinterpret_cast<int *>(&sh.verdict.state);
            for (int i = lane; i < (int) (sizeof(IcpState) / sizeof(int)); i += 32) dst[i] = src[i];
            if (lane < 4) sh.verdict.counts[lane] = __ldcg(tail.counts + lane);
            __syncwarp();
            if (lane == 0) frame_policy_decide(sh.verdict, tail.in);
            __syncwarp();
            frame_verdict_publish(sh.verdict, tail.dv, tail.hv, lane);
        }
    }
}

// Stand-alone exchange for the launch-per-step paths (solvers CERES / ROBUST: one per LM evaluation; GN with
// CTICP_PERSISTENT=0): acc ← Σ over ranks of acc, in place, one CTA.
__global__ void __launch_bounds__(256) k_peer_allreduce(PeerLinks links, double *__restrict__ acc, IcpState *st) {
    __shared__ double s_acc[kAcc];
    __shared__ unsigned int s_half[kMaxPeers * kPeerWords];
    __shared__ int s_ok;
    if (threadIdx.x < kAcc) s_acc[threadIdx.x] = acc[threadIdx.x];
    const unsigned int seq = *links.seq + 1;
    const bool ok = peer_allreduce(links, seq, s_acc, s_half, &s_ok);
    if (threadIdx.x < kAcc) acc[threadIdx.x] = s_acc[threadIdx.x];
    if (threadIdx.x == 0) {
        *links.seq = seq;
        if (!ok && st) {
            st->failed = 3;
            st->done = 1;
        }
    }
}

// multi-GPU tail: the all-reduced accumulator → GN step (one warp)
__global__ void k_gn_solve_acc(const double *__restrict__ acc_in, IcpState *st, GnParams P) {
    __shared__ SolveScratch s_solve;
    __shared__ double s_acc[kAcc];
    if (st->done) return;
    for (int i = threadIdx.x; i < kAcc; i += 32) s_acc[i] = acc_in[i];
    __syncwarp();
    warp_gn_solve(s_acc, s_solve, st, P, 0, nullptr, threadIdx.x);
}

// Neighbor lists for arbitrary queries (parity tests of the map search; ComputeNeighborhoods, map.h:532-540)
__global__ void __launch_bounds__(kGatherWarps * 32)
k_neighborhoods(GatherConfig G, const double *__restrict__ queries, int n, double *__restrict__ out_points,
                int *__restrict__ out_counts) {
    __shared__ KnnStage s_stage[kGatherWarps][64];
    __shared__ int s_stencil[kMaxStencil];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int *stencil = stencil_table_fill(s_stencil, G.r);
    __syncthreads();
    for (int i = blockIdx.x * kGatherWarps + w; i < n; i += gridDim.x * kGatherWarps) {
        const V3 q{queries[3 * i], queries[3 * i + 1], queries[3 * i + 2]};
        const QueryCtx ctx = make_query(q, G.L.res, lane);
        KnnEntry best;
        unsigned spts;
        const int cnt = warp_gather_knn(G, stencil, ctx, lane, s_stage[w], best, spts);
        if (lane == 0) out_counts[i] = cnt;
        if (lane < cnt) {
            const V3 rel = knn_rel_position(G, stencil, ctx, best);
            double *o = out_points + ((size_t) i * G.kmax + (cnt - 1 - lane)) * 3;   // farthest first
            o[0] = q.x + rel.x; o[1] = q.y + rel.y; o[2] = q.z + rel.z;
        }
        __syncwarp();
    }
}

// ComputeNeighborhoods(queries, radiuses, max_num_neighbors, true, sensor_location), map.h:434-447: per-query radius →
// per-query level and stencil; optional normal filter.
struct RadiusSearchLevels {
    int num_levels, filter;
    V3 sensor;
    MapLevel levels[CTICP_MAX_RESOLUTIONS];
};
__global__ void __launch_bounds__(kGatherWarps * 32)
k_radius_search(const RadiusSearchLevels *__restrict__ R, int kmax, const double *__restrict__ queries,
                const double *__restrict__ radiuses, int n, double *__restrict__ out_points, int *__restrict__ out_counts) {
    __shared__ KnnStage s_stage[kGatherWarps][64];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int i = blockIdx.x * kGatherWarps + w; i < n; i += gridDim.x * kGatherWarps) {
        const V3 q{queries[3 * i], queries[3 * i + 1], queries[3 * i + 2]};
        const double radius = radiuses[i];
        int it = 0;
        while (it < R->num_levels && R->levels[it].res <= radius) ++it;
        GatherConfig G;
        G.L = R->levels[it > 0 ? it - 1 : 0];
        G.r = (int) ceil(radius / G.L.res);
        G.radius2 = radius * radius;
        G.kmax = kmax;
        const QueryCtx ctx = make_query(q, G.L.res, lane);
        KnnEntry best;
        unsigned spts;
        int cnt;
        if (R->filter)
            cnt = warp_gather_knn<true>(G, nullptr, ctx, lane, s_stage[w], best, spts,
                                        V3{R->sensor.x - q.x, R->sensor.y - q.y, R->sensor.z - q.z});
        else
            cnt = warp_gather_knn<false>(G, nullptr, ctx, lane, s_stage[w], best, spts);
        if (lane == 0) out_counts[i] = cnt;
        if (lane < cnt) {
            const V3 rel = knn_rel_position(G, nullptr, ctx, best);
            double *o = out_points + ((size_t) i * kmax + (cnt - 1 - lane)) * 3;   // farthest first
            o[0] = q.x + rel.x; o[1] = q.y + rel.y; o[2] = q.z + rel.z;
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------------------------
void IcpSolver::SetPeerLinks(const PeerLinksHost &links) {
    links_host_ = links;
    peers_ready_ = links.world > 1 && links.seq != nullptr;
}
void IcpSolver::PreloadShardedKernels() {
    cudaFuncAttributes a;
    cudaFuncGetAttributes(&a, k_gn_persistent<true>);
    cudaFuncGetAttributes(&a, k_gn_persistent<false>);
    cudaFuncGetAttributes(&a, k_gn_iterate);
    cudaFuncGetAttributes(&a, k_peer_allreduce);
    cudaFuncGetAttributes(&a, k_gn_solve_acc);
    PreloadLmKernels();
    cudaGetLastError();
}
void IcpSolver::AllReduceAccumulator(void *nccl_comm, IcpState *d_state) {
    if (peers_ready_) {
        k_peer_allreduce<<<1, 256, 0, stream_>>>(PeerLinksOf(links_host_), d_acc_, d_state);
        launches_ += 1;
        return;
    }
    NcclAllReduceAccumulator(nccl_comm);
}

IcpSolver::IcpSolver(cudaStream_t stream) : stream_(stream) {
    if (const char *e = getenv("CTICP_PERSISTENT")) use_persistent_ = atoi(e) != 0;
    if (const char *e = getenv("CTICP_GN_KP_PER_CTA")) kp_per_cta_ = std::max(1, std::min(atoi(e), 32 * kGatherWarps));
    int dev = 0;
    cudaGetDevice(&dev);
    CT_CUDA_CHECK(cudaFuncSetAttribute(k_gn_iterate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) sizeof(GnShared)));
    CT_CUDA_CHECK(cudaFuncSetAttribute(k_gn_persistent<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) sizeof(GnShared)));
    CT_CUDA_CHECK(cudaFuncSetAttribute(k_gn_persistent<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) sizeof(GnShared)));
    cudaDeviceGetAttribute(&num_sms_, cudaDevAttrMultiProcessorCount, dev);
    CT_CUDA_CHECK(cudaMalloc(&d_sys_, sizeof(double) * 160));
    CT_CUDA_CHECK(cudaMalloc(&d_acc_, sizeof(double) * kAcc));
    CT_CUDA_CHECK(cudaMalloc(&d_ticket_, sizeof(unsigned int)));
    CT_CUDA_CHECK(cudaMemset(d_ticket_, 0, sizeof(unsigned int)));
    CT_CUDA_CHECK(cudaMalloc(&d_sync_words_, sizeof(unsigned int) * 128));   // two sets of (arrive, epoch), a 128-byte line each
    CT_CUDA_CHECK(cudaMemset(d_sync_words_, 0, sizeof(unsigned int) * 128));
    for (int i = 0; i < kMaxEvents; ++i) {
        CT_CUDA_CHECK(cudaEventCreate(&ev_begin_[i]));
        CT_CUDA_CHECK(cudaEventCreate(&ev_end_[i]));
    }
}
IcpSolver::~IcpSolver() {
    cudaFree(d_partials_);
    cudaFree(d_sys_);
    cudaFree(d_acc_);
    cudaFree(d_ticket_);
    cudaFree(d_sync_words_);
    FreeLmBuffers();
    for (int i = 0; i < kMaxEvents; ++i) {
        cudaEventDestroy(ev_begin_[i]);
        cudaEventDestroy(ev_end_[i]);
    }
}
void IcpSolver::EnsurePartials(int blocks) {
    if (blocks <= partial_blocks_) return;
    CT_CUDA_CHECK(cudaStreamSynchronize(stream_));
    cudaFree(d_partials_);
    CT_CUDA_CHECK(cudaMalloc(&d_partials_, sizeof(double) * kAcc * (size_t) blocks));
    partial_blocks_ = blocks;
}
GnParams IcpSolver::MakeParams(const DeviceMap &map, const cticp_icp_options &opt) const {
    GnParams P{};
    map.SearchParams(map.Options().default_radius, &P.level, &P.r);
    P.radius = map.Options().default_radius;
    P.kmax = opt.max_number_neighbors;
    P.kmin = opt.min_number_neighbors;
    P.max_dist_to_plane = opt.max_dist_to_plane_ct_icp;
    P.threshold_norm = opt.threshold_orientation_norm;
    P.shard_rank = 0;
    P.shard_world = 1;
    P.debug_flags = 0;
    if (const char *e = getenv("CTICP_DEBUG_FLAGS")) P.debug_flags = atoi(e);
    P.bucket_scale = (double) kSelBuckets / (P.radius * P.radius);
    P.kp_lo = kp_lo_;
    P.rigid_first = (opt.parametrization == CTICP_PARAM_SIMPLE && !opt.point_to_plane_with_distortion) ? 1 : 0;
    return P;
}
static int GatherBlocks(size_t k_hint, int max_blocks, int kp_per_cta) {
    // One CTA (kGatherWarps warps, 128 registers per thread) per SM. A keypoint set smaller than the machine is spread
    // thin — `kp_per_cta` keypoints per CTA, so each keypoint's warp has an SM sub-partition nearly to itself: the loop
    // is latency-bound there — until every SM has a CTA; beyond that the tiles widen (gn_gather_tiles).
    // k_hint is an ESTIMATE of the keypoint count (the exact count lives on the device): too small only widens the
    // tiles, too large only adds idle CTAs whose zero partials have to be summed.
    size_t want = (k_hint + kp_per_cta - 1) / kp_per_cta;
    return (int) std::max<size_t>(1, std::min(want, (size_t) max_blocks));
}

void IcpSolver::PrintWarpStamps(int iters) {
#ifdef CTICP_DEBUG_TIMERS
    if (!d_dbg_warp_ || dbg_warps_ <= 0) return;
    const int W = dbg_warps_;
    std::vector<unsigned long long> h((size_t) kDbgIters * W * kDbgSlots);
    CT_CUDA_CHECK(cudaMemcpy(h.data(), d_dbg_warp_, sizeof(unsigned long long) * h.size(), cudaMemcpyDeviceToHost));
    static const char *names[kDbgSlots] = {"A pose+voxel", "B gather+select", "C epilogue", "pose fetch", "fetch+tiles+row reduction", "barrier wait (per CTA)"};
    for (int it = 0; it < std::min(iters, kDbgIters); ++it) {
        fprintf(stderr, "[cticp] GN gather warps, iteration %d (SM cycles; %d warps):", it, W);
        for (int sl = 0; sl < kDbgSlots; ++sl) {
            std::vector<unsigned long long> v;
            for (int w = 0; w < W; ++w) {
                const unsigned long long x = h[((size_t) it * W + w) * kDbgSlots + sl];
                const unsigned long long busy = h[((size_t) it * W + w) * kDbgSlots + 4];
                if (sl == 5 ? (w < W / kGatherWarps) : busy != 0) v.push_back(x);
            }
            if (v.empty()) continue;
            std::sort(v.begin(), v.end());
            double mean = 0;
            for (auto x : v) mean += (double) x;
            mean /= (double) v.size();
            fprintf(stderr, "  %s mean %.0f p50 %llu p90 %llu max %llu;", names[sl], mean, v[v.size() / 2], v[v.size() * 9 / 10], v.back());
        }
        fprintf(stderr, "\n");
    }
#else
    (void) iters;
#endif
}

void IcpSolver::CollectGatherTiming() {
    for (int i = 0; i < ev_used_; ++i) {
        float ms = 0.f;
        // (the caller may have learnt the result from the frame verdict, which the device writes before — or, with
        // CTICP_TAIL_IN_KERNEL=1, from inside — the kernel this event follows)
        cudaEventSynchronize(ev_end_[i]);
        if (cudaEventElapsedTime(&ms, ev_begin_[i], ev_end_[i]) == cudaSuccess) gather_ms_ += ms;
    }
    ev_used_ = 0;
}

bool IcpSolver::EnqueueGaussNewton(const DeviceMap &map, const cticp_icp_options &opt, const float4 *d_keypoints,
                                   const int *d_num_keypoints, size_t k_upper, int num_iters, IcpState *d_state,
                                   int shard_rank, int shard_world, void *nccl_comm, const FrameTailArgs *tail) {
    if (opt.max_number_neighbors > 32 || opt.max_number_neighbors < 1)
        throw std::invalid_argument("max_number_neighbors must be in [1, 32]");
    GatherLaunch cfg;
    cfg.P = MakeParams(map, opt);
    cfg.P.shard_rank = shard_rank;
    cfg.P.shard_world = shard_world;
    cfg.G.L = map.Level(cfg.P.level);
    cfg.G.r = cfg.P.r;
    cfg.G.radius2 = cfg.P.radius * cfg.P.radius;
    cfg.G.kmax = cfg.P.kmax;
    const bool peers = nccl_comm && shard_world > 1 && peers_ready_;
    const size_t k_share = (k_upper + shard_world - 1) / shard_world + 16;
    if (use_persistent_ && (!nccl_comm || peers)) {
        // one cooperative launch for the whole loop; the grid must be co-resident (grid-wide barriers)
        void *kernel = peers ? (void *) k_gn_persistent<true> : (void *) k_gn_persistent<false>;
        int &coresident = max_coresident_[peers ? 1 : 0];
        if (coresident == 0) {
            int per_sm = 0;
            CT_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kGatherWarps * 32, sizeof(GnShared)));
            coresident = std::max(1, per_sm * num_sms_);
        }
        const int blocks = GatherBlocks(k_share, std::max(1, coresident - 1), kp_per_cta_);
        EnsurePartials(blocks + 1);
        int grid = std::min(blocks + 1, coresident);
        grid = std::max(grid, 2);
        const float4 *kp = d_keypoints;
        const int *nk = d_num_keypoints;
        double *parts = d_partials_;
        int iters = num_iters;
        PeerLinks links = peers ? PeerLinksOf(links_host_) : PeerLinks{};
#ifdef CTICP_DEBUG_TIMERS
        if (getenv("CTICP_DEBUG_TIMERS")) {
            const int warps = (grid - 1) * kGatherWarps;
            if (warps > dbg_warps_) {
                CT_CUDA_CHECK(cudaStreamSynchronize(stream_));
                cudaFree(d_dbg_warp_);
                CT_CUDA_CHECK(cudaMalloc(&d_dbg_warp_, sizeof(unsigned long long) * kDbgIters * warps * kDbgSlots));
            }
            dbg_warps_ = warps;
            CT_CUDA_CHECK(cudaMemsetAsync(d_dbg_warp_, 0, sizeof(unsigned long long) * kDbgIters * warps * kDbgSlots, stream_));
            cfg.P.dbg_warp = d_dbg_warp_;
        }
#endif
        LoopSync sync;
        sync.arrive = d_sync_words_ + 64 * sync_set_;
        sync.epoch = sync.arrive + 32;
        sync.next_arrive = d_sync_words_ + 64 * (sync_set_ ^ 1);
        sync.next_epoch = sync.next_arrive + 32;
        sync_set_ ^= 1;
        FrameTailArgs tail_args{};
        if (tail) tail_args = *tail;
        void *args[] = {&cfg, &kp, &nk, &d_state, &parts, &iters, &links, &sync, &tail_args};
        const bool timed = time_gather_ && ev_used_ < kMaxEvents;
        if (timed) cudaEventRecord(ev_begin_[ev_used_], stream_);
        CT_CUDA_CHECK(cudaLaunchCooperativeKernel(kernel, dim3(grid), dim3(kGatherWarps * 32), args, sizeof(GnShared), stream_));
        if (timed) cudaEventRecord(ev_end_[ev_used_++], stream_);
        gather_launches_ += 1;
        launches_ += 1;
        return tail != nullptr;
    }
    const int blocks = GatherBlocks(k_share, num_sms_, kp_per_cta_);
    EnsurePartials(blocks + 1);
    for (int it = 0; it < num_iters; ++it) {
        const bool timed = time_gather_ && ev_used_ < kMaxEvents;
        if (timed) cudaEventRecord(ev_begin_[ev_used_], stream_);
        k_gn_iterate<<<blocks, kGatherWarps * 32, sizeof(GnShared), stream_>>>(cfg, d_keypoints, d_num_keypoints, d_state,
                                                                              d_partials_, d_ticket_, nccl_comm ? 2 : 0, d_acc_, nullptr);
        if (timed) cudaEventRecord(ev_end_[ev_used_++], stream_);
        ++gather_launches_;
        launches_ += 1;
        if (nccl_comm) {
            AllReduceAccumulator(nccl_comm, d_state);   // in-place sum of d_acc_ over ranks (peer mailboxes, else NCCL)
            k_gn_solve_acc<<<1, 32, 0, stream_>>>(d_acc_, d_state, cfg.P);
            launches_ += 1;
        }
    }
    CT_CUDA_CHECK(cudaGetLastError());
    return false;
}

void IcpSolver::NormalEquations(const DeviceMap &map, const cticp_icp_options &opt, const float4 *d_keypoints,
                                const int *d_num_keypoints, size_t k_upper, IcpState *d_state, double *h_A144,
                                double *h_b12, int *h_n_used) {
    GatherLaunch cfg;
    cfg.P = MakeParams(map, opt);
    cfg.G.L = map.Level(cfg.P.level);
    cfg.G.r = cfg.P.r;
    cfg.G.radius2 = cfg.P.radius * cfg.P.radius;
    cfg.G.kmax = cfg.P.kmax;
    const int blocks = GatherBlocks(k_upper, num_sms_, kp_per_cta_);
    EnsurePartials(blocks);
    CT_CUDA_CHECK(cudaMemsetAsync(d_sys_, 0, sizeof(double) * 160, stream_));
    k_gn_iterate<<<blocks, kGatherWarps * 32, sizeof(GnShared), stream_>>>(cfg, d_keypoints, d_num_keypoints, d_state,
                                                                          d_partials_, d_ticket_, 1, d_acc_, d_sys_);
    launches_ += 1;
    double h[160];
    CT_CUDA_CHECK(cudaMemcpyAsync(h, d_sys_, sizeof(h), cudaMemcpyDeviceToHost, stream_));
    CT_CUDA_CHECK(cudaStreamSynchronize(stream_));
    for (int i = 0; i < 144; ++i) h_A144[i] = h[i];
    for (int i = 0; i < 12; ++i) h_b12[i] = h[144 + i];
    *h_n_used = (int) (h[156] + 0.5);
}

void IcpSolver::Neighborhoods(const DeviceMap &map, const double *d_queries, size_t n, int kmax, double *d_out_points,
                              int *d_out_counts) {
    if (kmax > 32 || kmax < 1) throw std::invalid_argument("max_num_neighbors must be in [1, 32]");
    GatherConfig G;
    int level, r;
    map.SearchParams(map.Options().default_radius, &level, &r);
    G.L = map.Level(level);
    G.r = r;
    G.radius2 = map.Options().default_radius * map.Options().default_radius;
    G.kmax = kmax;
    const int blocks = (int) std::max<size_t>(1, std::min((n + kGatherWarps - 1) / kGatherWarps, (size_t) num_sms_ * 2));
    k_neighborhoods<<<blocks, kGatherWarps * 32, 0, stream_>>>(G, d_queries, (int) n, d_out_points, d_out_counts);
    launches_ += 1;
    CT_CUDA_CHECK(cudaGetLastError());
}

void IcpSolver::RadiusSearch(const DeviceMap &map, const double *d_queries, const double *d_radiuses, size_t n, int kmax,
                             const double *sensor_location, double *d_out_points, int *d_out_counts) {
    if (kmax > 32 || kmax < 1) throw std::invalid_argument("max_num_neighbors must be in [1, 32]");
    RadiusSearchLevels R{};
    R.num_levels = map.NumLevels();
    R.filter = (sensor_location && map.Options().select_valid_normals_direction && map.HasNormals()) ? 1 : 0;
    if (sensor_location) R.sensor = V3{sensor_location[0], sensor_location[1], sensor_location[2]};
    for (int i = 0; i < R.num_levels; ++i) R.levels[i] = map.Level(i);
    RadiusSearchLevels *d_R = nullptr;
    CT_CUDA_CHECK(cudaMalloc(&d_R, sizeof(R)));
    CT_CUDA_CHECK(cudaMemcpyAsync(d_R, &R, sizeof(R), cudaMemcpyHostToDevice, stream_));
    const int blocks = (int) std::max<size_t>(1, std::min((n + kGatherWarps - 1) / kGatherWarps, (size_t) num_sms_ * 2));
    k_radius_search<<<blocks, kGatherWarps * 32, 0, stream_>>>(d_R, kmax, d_queries, d_radiuses, (int) n, d_out_points, d_out_counts);
    launches_ += 1;
    CT_CUDA_CHECK(cudaGetLastError());
    CT_CUDA_CHECK(cudaStreamSynchronize(stream_));
    cudaFree(d_R);
}

}  // namespace cticp
