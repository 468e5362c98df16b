// icp_lm.cu — solver CERES reproduced on the device as a Levenberg-Marquardt / robust-loss (IRLS) loop.
//
// Reference: DoRegisterCeres (src/ct_icp/ct_icp.cpp:460-706). Per ICP iteration:
//   k_lm_gather : one warp per keypoint — neighbor gather + normal/a2D (same device code as the GN path), emits one
//                 residual block per keypoint (:561-604): anchor point, normal, weight, alpha.
//   k_lm_select : GetProblem (:409-424): the first max_num_residuals valid blocks in keypoint order; seeds the LM state.
//   k_lm_eval   : half a warp per residual block; lane j evaluates the CTFunctor on dual numbers along tangent
//                 direction j (lm_functor.cuh), applies the loss function's Corrector, and the 12 partials are
//                 accumulated into JTJ (78) / JTr (12) / cost exactly like the GN accumulator.
//   k_lm_step   : ceres::Solve restated (TrustRegionMinimizer + LevenbergMarquardtStrategy, Ceres defaults except
//                 max_num_iterations = ls_max_num_iters): Jacobi scaling, LM diagonal, damped 12x12 solve, model cost
//                 change, candidate = Plus(x, delta); after the candidate has been evaluated: tolerances, step
//                 acceptance, trust-region radius update. The candidate is evaluated WITH its Jacobian, so an accepted
//                 step needs no second pass.
//   k_lm_finish : write the pose pair back, stop criterion of the ICP loop (:650-672).
// Every launch is enqueued up front; device-side flags turn the launches after convergence into no-ops.
#include <cstdio>
#include <cstdlib>

#include <cooperative_groups.h>

#include "engine.h"
#include "gather_select.cuh"
#include "icp.h"
#include "lm_functor.cuh"
#include "peer_exchange.cuh"
#include "small_solve.cuh"

namespace cticp {

constexpr int kLmWarps = 4;
constexpr int kAccCost = 91;   // Σ 1/2 rho(s) in the accumulator

struct LmParams {
    // ICP / neighborhood
    int r, level, kmax, kmin;
    double radius;
    double lambda_weight, lambda_neighborhood, power_planarity, max_dist_to_plane;
    int max_num_residuals, min_number_neighbors, num_iters_icp;
    int ncn;               // num_closest_neighbors (solver CERES, ct_icp.cpp:554,593-601): residual blocks per keypoint
    double bucket_scale;   // 32 / radius^2 (gather_select.cuh)
    double threshold_orientation_norm, threshold_translation_norm;
    // least squares
    LossParams loss;
    int ls_max_num_iters;
    int shard_rank, shard_world;
    // POSE_PARAMETRIZATION SIMPLE (motion compensation NONE / CONSTANT_VELOCITY / ITERATIVE, odometry.cpp:704-724): only the
    // end pose is optimised; `distortion` = point_to_plane_with_distortion (ITERATIVE)
    int simple, distortion;
    const float4 *kp_lo;   // residual plane of the keypoints (nullptr: float32-representable; load_raw, se3.cuh)
    // solver ROBUST (ct_icp.cpp:1180-1370)
    int robust, use_lines, use_barycenter;
    double threshold_linearity, threshold_planarity, outlier_distance, weight_neighborhood;
};

// std::pow(x, power_planarity) of the residual weights: the shipped configurations use 2.0 — x * x is that power correctly
// rounded (what glibc's pow returns for it too), without pow's ~300 instructions in the lane-per-keypoint phase
__device__ __forceinline__ double pow_weight(double x, double p) { return p == 2.0 ? x * x : pow(x, p); }

struct LmState {
    double x[14];        // current point: qb(4) qe(4) tb(3) te(3)   (Ceres program order of the parameter blocks)
    double cand[14];     // candidate point
    double best[14];     // TrustRegionMinimizer::parameters_ (lowest cost so far)
    double U[12][12];    // J^T J at x, unscaled
    double gu[12];       // J^T r at x, unscaled
    double scaling[12];  // jacobi_scaling
    double diagonal[12];
    double x_cost, minimum_cost, model_cost_change, radius, decrease_factor, x_norm, gradient_max_norm;
    int reuse_diagonal, iteration, done, step_is_successful, num_invalid, usable;
    int num_residuals, num_valid;   // this rank's share when the keypoints are sharded
    int num_residuals_global;       // residual blocks in the problem (all ranks)
    // ICP-loop bookkeeping (ct_icp.cpp:650-672)
    double prev_qb[4], prev_qe[4], prev_tb[3], prev_te[3];
    int outer_iter;
    // debug trace (CTICP_DEBUG_LM): one record per evaluated candidate
    // -DCTICP_DEBUG_TIMERS: SM cycles of the solver CTA per launch — [0] whole loop, [1] waiting for the residual assembly,
    // [2] GetProblem (selection), [3] waiting for an evaluation, [4] reduction of the partial rows, [5] minimizer step,
    // [6] the barriers behind a publish, [7] evaluations
    unsigned long long dbg_cycles[8];
    int trace_n;
    double trace[256][13];   // x_cost, candidate_cost, model_cost_change, relative_decrease, radius, flag
};

// DistanceBasedStrategy (neighborhood_strategy.h:95-146): the search radius — hence the map level and the stencil — is
// chosen per keypoint from its range, and the search filters on the per-voxel normals with sensor_location = the
// current end translation (ct_icp.cpp:571 passes &end_t).
struct DistanceStrategy {
    int num_levels, filter;
    double radius_min, radius_max, exponent;
    MapLevel levels[CTICP_MAX_RESOLUTIONS];
};

// ---------------------------------------------------------------------------------------------------------------
// Residual assembly, tiled like the GN gather (icp_gn.cu gn_gather_tiles): a warp owns W consecutive keypoints;
// lane j does keypoint j's scalar work (transform, per-keypoint radius, covariance → eigen → weight with its pow / exp,
// the 144-byte residual block) and the whole warp does the gather + k-nearest selection of each keypoint in turn.
constexpr int kLmTileMax = 16;
constexpr int kMaxNcn = 4;         // num_closest_neighbors supported (the reference's configurations all use 1)
constexpr int kRankTile = 4;
struct __align__(16) LmTile {
    SelScratch sel;
    double sums[kLmTileMax][14];   // n, stencil points, Σ rel (3), Σ rel rel^T (6), farthest kept (3)
    double ranked[kRankTile][kMaxNcn][3];    // num_closest_neighbors > 1 (tiles of at most kRankTile keypoints then): the head
                                             // of each keypoint's neighbor list, farthest first
};
__device__ __forceinline__ void lm_store_sums(double *o, const NeighborSums &s, unsigned spts, int need) {
    o[0] = __hiloint2double((int) spts, s.n);   // two integers in one slot: no int <-> double conversion (XU pipe, se3.cuh)
    if (s.n >= need) {
        o[2] = s.sx; o[3] = s.sy; o[4] = s.sz;
        o[5] = s.sxx; o[6] = s.sxy; o[7] = s.sxz; o[8] = s.syy; o[9] = s.syz; o[10] = s.szz;
        o[11] = s.fx; o[12] = s.fy; o[13] = s.fz;
    }
}
__device__ __forceinline__ NeighborSums lm_load_sums(const double *o) {
    NeighborSums s;
    s.n = __double2loint(o[0]);
    s.sx = o[2]; s.sy = o[3]; s.sz = o[4];
    s.sxx = o[5]; s.sxy = o[6]; s.sxz = o[7]; s.syy = o[8]; s.syz = o[9]; s.szz = o[10];
    s.fx = o[11]; s.fy = o[12]; s.fz = o[13]; s.fd2 = 0;
    return s;
}

// The tiles of a CTA's share of the keypoints: CTA `cta` of `num_ctas` owns a contiguous, balanced range; its
// `warps_per_cta` warps grab tiles of W consecutive keypoints from the shared-memory counter `next` (0 and visible on entry)
// until the range is exhausted — a warp whose keypoint has a sparse stencil takes the next one while a neighbour is still busy
// with a dense one. The blocks are written by keypoint index, so the result does not depend on who assembled them.
__device__ __forceinline__ int lm_tile_width(int span, int warps_per_cta) {
    if (span <= 2 * warps_per_cta) return 1;
    const int W = (span + warps_per_cta - 1) / warps_per_cta;
    return W < kLmTileMax ? W : kLmTileMax;
}
__device__ __forceinline__ int lm_grab_tile(int *next, int W, int lane) {
    int j0 = 0;
    if (lane == 0) j0 = atomicAdd(next, W);
    return __shfl_sync(0xffffffffu, j0, 0);
}

// One warp's share of the residual assembly of solver CERES (ct_icp.cpp:561-604).
// kCopy: the grouped k_lm_persistent's own copy (its G0 / P are in shared memory): the solo kernels' code stays as it is
template <bool kDB, bool kCopy = false>
__device__ __noinline__ void lm_gather_tiles(const GatherConfig &G0, const LmParams &P, const int *stencil,
                                                const float4 *__restrict__ keypoints, int K, const IcpState *st,
                                                ResidualBlock *__restrict__ blocks, unsigned long long *stats,
                                                const DistanceStrategy *__restrict__ D, LmTile &T, int cta, int num_ctas,
                                                int warps_per_cta, int *next, int lane) {
    const Q4 qb{__ldcg(&st->qb[0]), __ldcg(&st->qb[1]), __ldcg(&st->qb[2]), __ldcg(&st->qb[3])},
        qe{__ldcg(&st->qe[0]), __ldcg(&st->qe[1]), __ldcg(&st->qe[2]), __ldcg(&st->qe[3])};
    const V3 tb{__ldcg(&st->tb[0]), __ldcg(&st->tb[1]), __ldcg(&st->tb[2])}, te{__ldcg(&st->te[0]), __ldcg(&st->te[1]), __ldcg(&st->te[2])};
    const SlerpConsts sc{__ldcg(&st->slerp_theta), __ldcg(&st->slerp_inv_sin), __ldcg(&st->slerp_linear), __ldcg(&st->slerp_negate)};
    unsigned long long n_kp = 0, n_pts = 0;
    // keypoint-sharded mode (SURVEY §8e): this rank assembles the blocks of its contiguous chunk only
    const int kp_lo = (int) ((long long) K * P.shard_rank / P.shard_world);
    const int kp_hi = (int) ((long long) K * (P.shard_rank + 1) / P.shard_world);
    const int c_lo = kp_lo + (int) ((long long) (kp_hi - kp_lo) * cta / num_ctas);
    const int c_hi = kp_lo + (int) ((long long) (kp_hi - kp_lo) * (cta + 1) / num_ctas);
    int W = lm_tile_width(c_hi - c_lo, warps_per_cta);
    if (P.ncn > 1 && W > kRankTile) W = kRankTile;
    const int need = P.kmin > 5 ? P.kmin : 5;   // :574 ; neighborhood.h:227
    while (true) {
        const int t0 = c_lo + lm_grab_tile(next, W, lane);
        if (t0 >= c_hi) break;
        const int wt = (c_hi - t0) < W ? (c_hi - t0) : W;
        // ---- lane j: transform_keypoints() (ct_icp.cpp:516-531) and, for the distance-based strategy, this
        // keypoint's radius → map level + stencil (neighborhood_strategy.h:121-126, map.h:416-432)
        V3 p{0, 0, 0};
        int kx = 0, ky = 0, kz = 0, lvl = 0, rr = G0.r;
        double radius2 = G0.radius2, scale = P.bucket_scale;
        if (lane < wt) {
            const RawPoint kraw = load_raw(keypoints, P.kp_lo, t0 + lane);
            const V3 raw{kraw.x, kraw.y, kraw.z};
            // transform_keypoints (:516-531): interpolated pose unless SIMPLE without distortion (then the end pose)
            if (P.simple && !P.distortion)
                p = qrot(qnormalized(qe), raw) + te;
            else
                p = ct_transform_c(qb, tb, qe, te, kraw.alpha, raw, sc);
            double res = G0.L.res;
            if (kDB) {
                const double range = sqrt(raw.x * raw.x + raw.y * raw.y + raw.z * raw.z);
                const double a = pow(fmin(fabs(range), D->radius_max) / D->radius_max, D->exponent);
                const double radius = a * D->radius_max + (1 - a) * D->radius_min;
                int it = 0;
                while (it < D->num_levels && D->levels[it].res <= radius) ++it;
                lvl = it > 0 ? it - 1 : 0;
                res = D->levels[lvl].res;
                rr = (int) ceil(radius / res);
                radius2 = radius * radius;
                scale = (double) kSelBuckets / radius2;
            }
            kx = voxel_coord(p.x, res);
            ky = voxel_coord(p.y, res);
            kz = voxel_coord(p.z, res);
            confine_query(kx, ky, kz, rr);
        }
        // ---- all lanes: gather + selection, keypoint by keypoint
        for (int j = 0; j < wt; ++j) {
            const V3 q{__shfl_sync(0xffffffffu, p.x, j), __shfl_sync(0xffffffffu, p.y, j), __shfl_sync(0xffffffffu, p.z, j)};
            const int qx = __shfl_sync(0xffffffffu, kx, j), qy = __shfl_sync(0xffffffffu, ky, j),
                      qz = __shfl_sync(0xffffffffu, kz, j);
            GatherConfig G = G0;
            double sc_j = P.bucket_scale;
            if (kDB) {
                G.L = D->levels[__shfl_sync(0xffffffffu, lvl, j)];
                G.r = __shfl_sync(0xffffffffu, rr, j);
                G.radius2 = __shfl_sync(0xffffffffu, radius2, j);
                sc_j = __shfl_sync(0xffffffffu, scale, j);
            }
            NeighborSums s;
            unsigned spts = 0;
            double *ranked = P.ncn > 1 ? &T.ranked[j][0][0] : nullptr;
            if (kDB && D->filter)
                warp_gather_sums<true>(G, sc_j, stencil, q, qx, qy, qz, need, lane, T.sel, s, spts,
                                       V3{te.x - q.x, te.y - q.y, te.z - q.z}, nullptr, ranked, P.ncn);
            else
                warp_gather_sums<false>(G, sc_j, stencil, q, qx, qy, qz, need, lane, T.sel, s, spts, V3{0, 0, 0}, nullptr,
                                        ranked, P.ncn);
            if (lane == 0) lm_store_sums(T.sums[j], s, spts, need);
        }
        __syncwarp();
        // ---- lane j: the residual block (:574-604)
        if (lane < wt) {
            const int kp = t0 + lane;
            const NeighborSums mine = lm_load_sums(T.sums[lane]);
            n_kp += 1;
            n_pts += (unsigned long long) (unsigned) __double2hiint(T.sums[lane][0]);
            if (mine.n >= need) {
                const NeighborhoodDesc nd = describe_from_sums(mine);
                // (the normal flip test at :578 is a no-op: BeginTr - BeginTr)
                double weight = pow_weight(nd.a2D, P.power_planarity);
                const double far_dist = sqrt(nd.far_rel.x * nd.far_rel.x + nd.far_rel.y * nd.far_rel.y + nd.far_rel.z * nd.far_rel.z);
                weight = P.lambda_weight * weight +
                         P.lambda_neighborhood * exp(-far_dist / (P.max_dist_to_plane * P.min_number_neighbors));   // :582-587
                ResidualBlock rb;
                rb.ref[0] = p.x + nd.far_rel.x; rb.ref[1] = p.y + nd.far_rel.y; rb.ref[2] = p.z + nd.far_rel.z;   // points[0]
                rb.normal[0] = nd.normal.x; rb.normal[1] = nd.normal.y; rb.normal[2] = nd.normal.z;
                rb.weight = weight;
                const RawPoint kraw = load_raw(keypoints, P.kp_lo, t0 + lane);
                rb.alpha = kraw.alpha;
                V3 rawc{kraw.x, kraw.y, kraw.z};
                if (P.simple && P.distortion) {
                    // ICPOptimizationBuilder::DistortFrame (:198-215): the raw point in the frame of the END pose
                    const V3 w = ct_transform_c(qb, tb, qe, te, kraw.alpha, rawc, sc);
                    const Q4 qi = qinverse(qe);
                    rawc = qrot(qi, w) + (-1.0) * qrot(qi, te);
                }
                rb.raw[0] = rawc.x; rb.raw[1] = rawc.y; rb.raw[2] = rawc.z;
                rb.valid = 1;
                for (int i = 0; i < 6; ++i) rb.info[i] = 0.0;
                rb.kind = kResPlane | (P.simple ? kResSimple : 0);
                blocks[(size_t) P.ncn * kp] = rb;
                // num_closest_neighbors > 1 (ct_icp.cpp:593-601): the same normal, weight and raw point against the next
                // neighbors of the list (farthest first), block ncn * k + i
                for (int i = 1; i < P.ncn; ++i) {
                    const double *r = T.ranked[lane][i];
                    rb.ref[0] = p.x + r[0]; rb.ref[1] = p.y + r[1]; rb.ref[2] = p.z + r[2];
                    blocks[(size_t) P.ncn * kp + i] = rb;
                }
            } else {
                for (int i = 0; i < P.ncn; ++i) blocks[(size_t) P.ncn * kp + i].valid = 0;
            }
        }
        __syncwarp();
    }
    n_kp = __reduce_add_sync(0xffffffffu, (unsigned) n_kp);
    {
        unsigned long long t = n_pts;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        n_pts = t;
    }
    if (lane == 0 && n_kp) {
        atomicAdd(&stats[0], n_kp);
        atomicAdd(&stats[1], n_pts);
    }
}

template <bool kDB>
__global__ void __launch_bounds__(kLmWarps * 32)
k_lm_gather(GatherConfig G0, LmParams P, const float4 *__restrict__ keypoints, const int *__restrict__ d_num_keypoints,
            const IcpState *__restrict__ st, ResidualBlock *__restrict__ blocks, unsigned long long *stats,
            const DistanceStrategy *__restrict__ D) {
    __shared__ LmTile s_tile[kLmWarps];
    __shared__ int s_stencil[kMaxStencil];
    __shared__ int s_next;
    if (st->done) return;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int *stencil = kDB ? nullptr : stencil_table_fill(s_stencil, G0.r);
    if (threadIdx.x == 0) s_next = 0;
    __syncthreads();
    lm_gather_tiles<kDB>(G0, P, stencil, keypoints, *d_num_keypoints, st, blocks, stats, D, s_tile[w],
                         (int) blockIdx.x, (int) gridDim.x, kLmWarps, &s_next, lane);
}

// Solver ROBUST's per-keypoint assembly (ct_icp.cpp:1229-1289): same gather, the neighborhood is classified planar /
// linear / other and yields a point-to-plane / point-to-line / point-to-distribution block. `classes` holds
// slam::NEIGHBORHOOD_TYPE per keypoint ACROSS the ICP iterations: the reference keeps its `neighborhoods` vector alive
// (:1214) and ClassifyNeighborhood (neighborhood.h:268-282) leaves the previous class in place when neither threshold
// is passed.
template <bool kCopy = false>   // (as lm_gather_tiles)
__device__ __noinline__ void rb_gather_tiles(const GatherConfig &G, const LmParams &P, const int *stencil,
                                                const float4 *__restrict__ keypoints, int K, const IcpState *st,
                                                ResidualBlock *__restrict__ blocks, unsigned char *__restrict__ classes,
                                                unsigned long long *stats, LmTile &T, int cta, int num_ctas,
                                                int warps_per_cta, int *next, int lane) {
    enum { NONE = 0, LINEAR = 1, PLANAR = 2, VOLUMIC = 3 };
    const Q4 qb{__ldcg(&st->qb[0]), __ldcg(&st->qb[1]), __ldcg(&st->qb[2]), __ldcg(&st->qb[3])},
        qe{__ldcg(&st->qe[0]), __ldcg(&st->qe[1]), __ldcg(&st->qe[2]), __ldcg(&st->qe[3])};
    const V3 tb{__ldcg(&st->tb[0]), __ldcg(&st->tb[1]), __ldcg(&st->tb[2])}, te{__ldcg(&st->te[0]), __ldcg(&st->te[1]), __ldcg(&st->te[2])};
    const SlerpConsts sc{__ldcg(&st->slerp_theta), __ldcg(&st->slerp_inv_sin), __ldcg(&st->slerp_linear), __ldcg(&st->slerp_negate)};
    unsigned long long n_kp = 0, n_pts = 0;
    // keypoint-sharded mode (SURVEY §8e): this rank assembles the blocks of its contiguous chunk only
    const int kp_lo = (int) ((long long) K * P.shard_rank / P.shard_world);
    const int kp_hi = (int) ((long long) K * (P.shard_rank + 1) / P.shard_world);
    const int c_lo = kp_lo + (int) ((long long) (kp_hi - kp_lo) * cta / num_ctas);
    const int c_hi = kp_lo + (int) ((long long) (kp_hi - kp_lo) * (cta + 1) / num_ctas);
    const int W = lm_tile_width(c_hi - c_lo, warps_per_cta);
    const int need = P.kmin;   // :1238 (kmin >= 5 is enforced by the host, so the neighborhood is always describable)
    const double inv_res = 1.0 / G.L.res;
    while (true) {
        const int t0 = c_lo + lm_grab_tile(next, W, lane);
        if (t0 >= c_hi) break;
        const int wt = (c_hi - t0) < W ? (c_hi - t0) : W;
        V3 p{0, 0, 0};
        int kx = 0, ky = 0, kz = 0;
        if (lane < wt) {
            const RawPoint kraw = load_raw(keypoints, P.kp_lo, t0 + lane);
            p = ct_transform_c(qb, tb, qe, te, kraw.alpha, V3{kraw.x, kraw.y, kraw.z}, sc);   // TransformKeyPoints, :1373-1393
            kx = query_voxel_coord(p.x, G.L.res, inv_res);
            ky = query_voxel_coord(p.y, G.L.res, inv_res);
            kz = query_voxel_coord(p.z, G.L.res, inv_res);
            confine_query(kx, ky, kz, G.r);
        }
        for (int j = 0; j < wt; ++j) {
            const V3 q{__shfl_sync(0xffffffffu, p.x, j), __shfl_sync(0xffffffffu, p.y, j), __shfl_sync(0xffffffffu, p.z, j)};
            const int qx = __shfl_sync(0xffffffffu, kx, j), qy = __shfl_sync(0xffffffffu, ky, j),
                      qz = __shfl_sync(0xffffffffu, kz, j);
            NeighborSums s;
            unsigned spts = 0;
            warp_gather_sums<false>(G, P.bucket_scale, stencil, q, qx, qy, qz, need, lane, T.sel, s, spts);
            if (lane == 0) lm_store_sums(T.sums[j], s, spts, need);
        }
        __syncwarp();
        if (lane < wt) {
            const int kp = t0 + lane;
            const NeighborSums mine = lm_load_sums(T.sums[lane]);
            n_kp += 1;
            n_pts += (unsigned long long) (unsigned) __double2hiint(T.sums[lane][0]);
            int valid = 0;
            if (mine.n >= need) {
                const NeighborhoodDescFull nd = describe_full_from_sums(mine);
                int cls = classes[kp];
                if (nd.planarity > P.threshold_planarity) cls = PLANAR;
                else if (nd.linearity > P.threshold_linearity) cls = LINEAR;
                if (!P.use_lines && cls == LINEAR) cls = P.threshold_planarity < nd.planarity ? PLANAR : VOLUMIC;   // :1243-1248
                double weight;
                if (cls == LINEAR) weight = pow_weight(fabs(nd.linearity), P.power_planarity);
                else if (cls == PLANAR) weight = pow_weight(fabs(nd.planarity), P.power_planarity);
                else weight = P.weight_neighborhood;
                const V3 d = P.use_barycenter ? nd.mean_rel : nd.far_rel;   // point - world_point
                double distance;
                int kind = kResDistribution;
                if (cls == LINEAR) {
                    V3 u = nd.line;
                    const double z = dot(u, u);
                    if (z > 0) u = (1.0 / sqrt(z)) * u;
                    const V3 c = cross(d, u);
                    distance = sqrt(dot(c, c));
                    kind = kResLine;
                } else if (cls == PLANAR) {
                    distance = fabs(dot(d, nd.normal));
                    kind = kResPlane;
                } else {
                    distance = sqrt(dot(d, d));
                }
                classes[kp] = (unsigned char) cls;
                if (distance < P.outlier_distance) {
                    ResidualBlock rb;
                    rb.ref[0] = p.x + d.x; rb.ref[1] = p.y + d.y; rb.ref[2] = p.z + d.z;
                    const V3 dir = kind == kResLine ? nd.line : nd.normal;
                    rb.normal[0] = dir.x; rb.normal[1] = dir.y; rb.normal[2] = dir.z;
                    rb.weight = weight;
                    const RawPoint kraw = load_raw(keypoints, P.kp_lo, t0 + lane);
                    rb.alpha = kraw.alpha;
                    rb.raw[0] = kraw.x; rb.raw[1] = kraw.y; rb.raw[2] = kraw.z;
                    rb.valid = 1;
                    rb.kind = kind;
                    if (kind == kResDistribution) {
                        // (covariance + 0.05 I).inverse(), cost_functions.h:147-158 (Eigen's cofactor inverse)
                        const double m00 = nd.cov[0] + 0.05, m01 = nd.cov[1], m02 = nd.cov[2], m11 = nd.cov[3] + 0.05,
                                     m12 = nd.cov[4], m22 = nd.cov[5] + 0.05;
                        const double c00 = m11 * m22 - m12 * m12, c01 = m12 * m02 - m01 * m22, c02 = m01 * m12 - m11 * m02;
                        const double c11 = m22 * m00 - m02 * m02, c12 = m02 * m01 - m12 * m00, c22 = m00 * m11 - m01 * m01;
                        const double invdet = 1.0 / (c00 * m00 + c01 * m01 + c02 * m02);
                        rb.info[0] = c00 * invdet; rb.info[1] = c01 * invdet; rb.info[2] = c02 * invdet;
                        rb.info[3] = c11 * invdet; rb.info[4] = c12 * invdet; rb.info[5] = c22 * invdet;
                    } else {
                        for (int i = 0; i < 6; ++i) rb.info[i] = 0.0;
                    }
                    blocks[kp] = rb;
                    valid = 1;
                }
            }
            if (!valid) blocks[kp].valid = 0;
        }
        __syncwarp();
    }
    n_kp = __reduce_add_sync(0xffffffffu, (unsigned) n_kp);
    {
        unsigned long long t = n_pts;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        n_pts = t;
    }
    if (lane == 0 && n_kp) {
        atomicAdd(&stats[0], n_kp);
        atomicAdd(&stats[1], n_pts);
    }
}

__global__ void __launch_bounds__(kLmWarps * 32)
k_rb_gather(GatherConfig G, LmParams P, const float4 *__restrict__ keypoints, const int *__restrict__ d_num_keypoints,
            const IcpState *__restrict__ st, ResidualBlock *__restrict__ blocks, unsigned char *__restrict__ classes,
            unsigned long long *stats) {
    __shared__ LmTile s_tile[kLmWarps];
    __shared__ int s_stencil[kMaxStencil];
    __shared__ int s_next;
    if (st->done) return;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int *stencil = stencil_table_fill(s_stencil, G.r);
    if (threadIdx.x == 0) s_next = 0;
    __syncthreads();
    rb_gather_tiles(G, P, stencil, keypoints, *d_num_keypoints, st, blocks, classes, stats, s_tile[w],
                    (int) blockIdx.x, (int) gridDim.x, kLmWarps, &s_next, lane);
}

// GetProblem (ct_icp.cpp:409-424) + seeding of the LM state for this ICP iteration. One CTA.
// Sharded: launched twice. mode 1 counts this rank's valid blocks into counts[rank] (the vector is then summed over the
// ranks = all-gather); mode 0 selects with the global rank of each block = (valid blocks of lower ranks) + local rank,
// so the union over ranks is exactly the first max_num_residuals valid blocks in keypoint order.
struct LmSelectScratch {
    int warp[32];
    int carry;
};
// Called by ALL threads of one CTA (any multiple of 32 up to 1024 threads).
__device__ __forceinline__ void lm_select_device(const LmParams &P, int mode, int K, const ResidualBlock *__restrict__ blocks,
                                                 int *__restrict__ sel_idx, IcpState *st, LmState *lm,
                                                 const unsigned long long *stats, double *__restrict__ counts,
                                                 LmSelectScratch &sc) {
    int *s_warp = sc.warp;
    int &s_carry = sc.carry;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5, nthreads = blockDim.x;
    if (tid == 0) s_carry = 0;
    if (tid < 32) s_warp[tid] = 0;
    __syncthreads();
    const int limit = P.max_num_residuals > 0 ? P.max_num_residuals : 0x7fffffff;
    // (block slots ncn * k + i of this rank's keypoints, in slot order: builder.SetResidualBlock, ct_icp.cpp:598)
    const int kp_lo = P.ncn * (int) ((long long) K * P.shard_rank / P.shard_world);
    const int kp_hi = P.ncn * (int) ((long long) K * (P.shard_rank + 1) / P.shard_world);
    int before = 0, total_valid = -1;   // valid blocks on lower ranks / on all ranks
    if (P.shard_world > 1 && mode == 0) {
        total_valid = 0;
        for (int r = 0; r < P.shard_world; ++r) {
            const int c = (int) (counts[r] + 0.5);
            if (r < P.shard_rank) before += c;
            total_valid += c;
        }
    }
    for (int base = kp_lo; base < kp_hi; base += nthreads) {
        const int k = base + tid;
        const int v = (k < kp_hi) ? (blocks[k].valid != 0) : 0;
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        if (lane == 31) s_warp[w] = incl;
        __syncthreads();
        if (w == 0) {
            int ws = lane < (nthreads >> 5) ? s_warp[lane] : 0;   // (entries beyond the CTA's warps hold last round's totals)
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, ws, o);
                if (lane >= o) ws += y;
            }
            s_warp[lane] = ws;
        }
        __syncthreads();
        const int carry = s_carry;
        const int rank = carry + (w > 0 ? s_warp[w - 1] : 0) + incl - v;
        if (mode == 0 && v && before + rank < limit) sel_idx[rank] = k;
        __syncthreads();
        if (tid == nthreads - 1) s_carry = carry + s_warp[31];
        __syncthreads();
    }
    if (mode == 1) {
        if (tid < P.shard_world) counts[tid] = (tid == P.shard_rank) ? (double) s_carry : 0.0;
        return;
    }
    if (tid == 0) {
        const int num_valid = s_carry;
        if (total_valid < 0) total_valid = num_valid;
        const int R = total_valid < limit ? total_valid : limit;                       // the whole problem
        int R_local = limit - before;                                                   // this rank's share of it
        R_local = R_local < 0 ? 0 : (R_local < num_valid ? R_local : num_valid);
        lm->num_valid = num_valid;
        lm->num_residuals = R_local;
        lm->num_residuals_global = R;
        st->n_used = R;
        st->stat_keypoint_iters = stats[0];
        st->stat_stencil_points = stats[1];
        if (R < P.min_number_neighbors) {   // ct_icp.cpp:617 (sic: compared with min_number_neighbors)
            st->failed = 1;
            st->done = 1;
            lm->done = 1;
            return;
        }
        // parameter blocks in Ceres program order: begin_quat, end_quat, begin_t, end_t (ct_icp.cpp:229-232)
        for (int d = 0; d < 4; ++d) { lm->x[d] = st->qb[d]; lm->x[4 + d] = st->qe[d]; }
        for (int d = 0; d < 3; ++d) { lm->x[8 + d] = st->tb[d]; lm->x[11 + d] = st->te[d]; }
        lm->done = 0;
        lm->usable = 1;
        lm->iteration = 0;
        lm->radius = 1e4;                 // initial_trust_region_radius
        lm->decrease_factor = 2.0;
        lm->reuse_diagonal = 0;
        lm->num_invalid = 0;
        lm->minimum_cost = 1.7976931348623157e308;
        lm->step_is_successful = 1;
    }
}
__global__ void __launch_bounds__(1024)
k_lm_select(LmParams P, int mode, const int *__restrict__ d_num_keypoints, const ResidualBlock *__restrict__ blocks,
            int *__restrict__ sel_idx, IcpState *st, LmState *lm, const unsigned long long *stats,
            double *__restrict__ counts) {
    __shared__ LmSelectScratch sc;
    if (st->done) return;
    lm_select_device(P, mode, *d_num_keypoints, blocks, sel_idx, st, lm, stats, counts, sc);
}

// `half_index` / `halves_total`: this half-warp's index among all evaluating half-warps of the launch. s_u / s_acc: this
// CTA's scratch, one row per half-warp (hw = local half-warp index). Writes the CTA's sum to `row_out` (kAcc doubles).
// Called by ALL threads of the CTA.
template <int kHalves, bool kCopy = false>   // (kCopy as lm_gather_tiles)
__device__ __noinline__ void lm_eval_device(const LmParams &P, int which, const ResidualBlock *__restrict__ blocks,
                                               const int *__restrict__ sel_idx, const IcpState *st, const LmState *lm,
                                               double (*s_u)[16], double (*s_acc)[kAcc], int half_index, int halves_total,
                                               double *__restrict__ row_out) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int hl = lane & 15, half = lane >> 4, hw = w * 2 + half;
    const unsigned hmask = half ? 0xffff0000u : 0x0000ffffu;
    double acc[6] = {0, 0, 0, 0, 0, 0};   // entries hl + 16 m of [JTJ upper | JTr]
    double cost = 0;
    const bool active = !__ldcg(&st->done) && !__ldcg(&lm->done);
    if (active) {
        const double *x = which ? lm->cand : lm->x;
        double qb[4], qe[4], tb[3], te[3];
#pragma unroll
        for (int d = 0; d < 4; ++d) { qb[d] = __ldcg(x + d); qe[d] = __ldcg(x + 4 + d); }
#pragma unroll
        for (int d = 0; d < 3; ++d) { tb[d] = __ldcg(x + 8 + d); te[d] = __ldcg(x + 11 + d); }
        const int R = __ldcg(&lm->num_residuals);
        int pi[6], pj[6];
#pragma unroll
        for (int m = 0; m < 6; ++m) {
            const int e = hl + 16 * m;
            pi[m] = e < kAccUsed ? c_pair_i[e] : 0;
            pj[m] = e < kAccUsed ? c_pair_j[e] : 0;
        }
        for (int r = half_index; r < R; r += halves_total) {
            const ResidualBlock rb = blocks[__ldcg(sel_idx + r)];
            const Dual res = P.robust ? ct_residual<true>(rb, qb, qe, tb, te, hl) : ct_residual<false>(rb, qb, qe, tb, te, hl);
            const double s = res.a * res.a;
            double rs = 1.0, js = 1.0;
            if (P.loss.type != 0) {
                double rho[3];
                loss_evaluate(P.loss, s, rho);
                if (hl == 0) cost += 0.5 * rho[0];
                corrector_1d(s, rho, rs, js);
            } else if (hl == 0) {
                cost += 0.5 * s;
            }
            if (hl < 12) s_u[hw][hl] = js * res.d;
            if (hl == 12) s_u[hw][12] = rs * res.a;
            __syncwarp(hmask);
#pragma unroll
            for (int m = 0; m < 6; ++m)
                if (hl + 16 * m < kAccUsed) acc[m] += s_u[hw][pi[m]] * s_u[hw][pj[m]];
            __syncwarp(hmask);
        }
    }
    for (int m = 0; m < 6; ++m) s_acc[hw][hl + 16 * m] = (hl + 16 * m < kAccUsed) ? acc[m] : 0.0;
    __syncwarp();
    if (hl == 0) {
        s_acc[hw][kAccUsed] = 0;
        s_acc[hw][kAccCost] = cost;
    }
    __syncthreads();
    if (threadIdx.x < kAcc) {
        double s = 0;
#pragma unroll
        for (int h = 0; h < kHalves; ++h) s += s_acc[h][threadIdx.x];
        __stcg(row_out + threadIdx.x, s);
    }
}

// residual evaluation at lm->x (which = 0) or lm->cand (which = 1): half a warp per residual block
__global__ void __launch_bounds__(kLmWarps * 32)
k_lm_eval(LmParams P, int which, const ResidualBlock *__restrict__ blocks, const int *__restrict__ sel_idx,
          const IcpState *__restrict__ st, const LmState *__restrict__ lm, double *__restrict__ partials) {
    __shared__ double s_u[kLmWarps * 2][16];
    __shared__ double s_acc[kLmWarps * 2][kAcc];
    const int hw = (threadIdx.x >> 5) * 2 + ((threadIdx.x & 31) >> 4);
    lm_eval_device<kLmWarps * 2>(P, which, blocks, sel_idx, st, lm, s_u, s_acc, blockIdx.x * kLmWarps * 2 + hw,
                                 gridDim.x * kLmWarps * 2, partials + (size_t) blockIdx.x * kAcc);
}

// sharded mode: fold this rank's evaluation partials into one accumulator row for the all-reduce
__global__ void __launch_bounds__(128)
k_lm_reduce(const double *__restrict__ partials, int nblocks, double *__restrict__ acc) {
    if (threadIdx.x >= kAcc) return;
    double s = 0;
    for (int b = 0; b < nblocks; ++b) s += partials[(size_t) b * kAcc + threadIdx.x];
    acc[threadIdx.x] = s;
}

// ---- the minimizer ------------------------------------------------------------------------------------------
// what the regularisers read of the registration state: constant over a frame, kept next to the minimizer's scratch so
// that the serial step never waits for global memory (each of its ~25 reads of `st` was a dependent L2 round trip)
struct LmRegs {
    int has_motion_model;
    double beta_location, beta_orientation, beta_cv, beta_small;
    double prev_tb[3], prev_te[3], prev_qe[4];
};
__device__ __forceinline__ void lm_load_regs(LmRegs &r, const IcpState *st, int lane) {   // one warp; independent loads
    if (lane == 0) r.has_motion_model = st->has_motion_model;
    if (lane == 1) r.beta_location = st->beta_location;
    if (lane == 2) r.beta_orientation = st->beta_orientation;
    if (lane == 3) r.beta_cv = st->beta_cv;
    if (lane == 4) r.beta_small = st->beta_small;
    if (lane >= 5 && lane < 8) r.prev_tb[lane - 5] = st->prev_tb[lane - 5];
    if (lane >= 8 && lane < 11) r.prev_te[lane - 8] = st->prev_te[lane - 8];
    if (lane >= 11 && lane < 15) r.prev_qe[lane - 11] = st->prev_qe[lane - 11];
    __syncwarp();
}

struct LmScratch {
    LmRegs regs;
    double acc[kAcc];
    double U[12][12], gu[12];
    double cost;
    double step[12], delta[12];
    double neg[12], proj[14];   // -gradient and x ⊞ (-gradient) of the gradient-norm test
    SolveScratch solve;
    int flag;
};

// regularisers (PreviousFrameMotionModel::AddConstraintsToCeresProblem, motion_model.cpp:12-61), no loss function:
// adds their J^T J, J^T r and cost at the point p to (U, gu, cost). Serial (lane 0).
__device__ void add_regularisers(const LmRegs *st, int R, const double *p, double U[12][12], double gu[12], double &cost) {
    if (!st->has_motion_model) return;
    const double *qb = p, *tb = p + 8, *te = p + 11;
    if (st->beta_location > 0.) {   // LocationConsistencyFunctor on begin_t
        const double w = sqrt(R * st->beta_location);
        for (int k = 0; k < 3; ++k) {
            const double res = w * (tb[k] - st->prev_te[k]);
            cost += 0.5 * res * res;
            U[6 + k][6 + k] += w * w;
            gu[6 + k] += w * res;
        }
    }
    if (st->beta_orientation > 0.) {   // OrientationConsistencyFunctor on begin_quat
        const double w = sqrt(R * st->beta_orientation);
        const double s = qb[0] * st->prev_qe[0] + qb[1] * st->prev_qe[1] + qb[2] * st->prev_qe[2] + qb[3] * st->prev_qe[3];
        const double res = w * (1.0 - s * s);
        cost += 0.5 * res * res;
        double J[3];
        for (int k = 0; k < 3; ++k) {
            double col[4];
            quat_plus_column(qb, k, col);
            double g = 0;
            for (int c = 0; c < 4; ++c) g += -2.0 * w * s * st->prev_qe[c] * col[c];
            J[k] = g;
        }
        for (int a = 0; a < 3; ++a) {
            gu[a] += J[a] * res;
            for (int b = 0; b < 3; ++b) U[a][b] += J[a] * J[b];
        }
    }
    if (st->beta_cv > 0.) {   // ConstantVelocityFunctor(begin_t, end_t)
        const double w = sqrt(R * st->beta_cv);
        for (int k = 0; k < 3; ++k) {
            const double prev_velocity = st->prev_te[k] - st->prev_tb[k];
            const double res = w * (te[k] - tb[k] - prev_velocity);
            cost += 0.5 * res * res;
            U[6 + k][6 + k] += w * w;
            U[9 + k][9 + k] += w * w;
            U[6 + k][9 + k] -= w * w;
            U[9 + k][6 + k] -= w * w;
            gu[6 + k] += -w * res;
            gu[9 + k] += w * res;
        }
    }
    if (st->beta_small > 0.) {   // SmallVelocityFunctor
        const double w = sqrt(R * st->beta_small);
        for (int k = 0; k < 3; ++k) {
            const double res = w * (tb[k] - te[k]);
            cost += 0.5 * res * res;
            U[6 + k][6 + k] += w * w;
            U[9 + k][9 + k] += w * w;
            U[6 + k][9 + k] -= w * w;
            U[9 + k][6 + k] -= w * w;
            gu[6 + k] += w * res;
            gu[9 + k] += -w * res;
        }
    }
}

__device__ void lm_plus(const double *x, const double *delta, double *out) {
    const Q4 qb = quat_plus(Q4{x[0], x[1], x[2], x[3]}, delta[0], delta[1], delta[2]);
    const Q4 qe = quat_plus(Q4{x[4], x[5], x[6], x[7]}, delta[3], delta[4], delta[5]);
    out[0] = qb.x; out[1] = qb.y; out[2] = qb.z; out[3] = qb.w;
    out[4] = qe.x; out[5] = qe.y; out[6] = qe.z; out[7] = qe.w;
    for (int k = 0; k < 3; ++k) out[8 + k] = x[8 + k] + delta[6 + k];
    for (int k = 0; k < 3; ++k) out[11 + k] = x[11 + k] + delta[9 + k];
}
// norm over the problem's parameter blocks: all 14 numbers, or end_quat + end_t with parametrization SIMPLE
__device__ double norm14(const double *v, int simple = 0) {
    double s = 0;
    for (int i = 0; i < 14; ++i)
        if (!simple || (i >= 4 && i < 8) || i >= 11) s += v[i] * v[i];
    return sqrt(s);
}

// the minimizer step is bound by instruction fetch (see small_solve.cuh): the compact shared-memory form of the solve
__device__ __forceinline__ void lm_solve12(SolveScratch &S, int lane) { warp_ldlt_solve12_compact(S, lane); }

// phase 0: the accumulator holds the evaluation at lm->x (start of ceres::Solve: IterationZero).
// phase 1: the accumulator holds the evaluation at lm->cand.
// One warp; the 12x12 solves are warp-collective, the scalar logic runs on lane 0.
// kPeers (multi-GPU): the evaluation is the sum over ranks — the exchange (peer_exchange.cuh) happens here, between
// the reduction of this rank's partials and the minimizer step, so a sharded LM evaluation costs the same two launches
// as a single-GPU one. The early return below is taken by all ranks together (done flags derive from identical sums),
// so the ranks' exchange counters stay in step.
// The minimizer step on the evaluation held in S.acc (already reduced over this rank's CTAs and, when sharded, over the
// ranks). ONE WARP; the 12x12 solves are warp-collective, the scalar logic runs on lane 0.
// x ⊞ delta for the two quaternion blocks (lanes 0, 1) and the six translation components (lanes 2..7) at once
__device__ __forceinline__ void lm_plus_warp(const double *x, const double *delta, double *out, int lane) {
    if (lane < 2) {
        const double *q = x + 4 * lane, *d = delta + 3 * lane;
        const Q4 r = quat_plus(Q4{q[0], q[1], q[2], q[3]}, d[0], d[1], d[2]);
        double *o = out + 4 * lane;
        o[0] = r.x; o[1] = r.y; o[2] = r.z; o[3] = r.w;
    } else if (lane < 8) {
        const int k = lane - 2;
        out[8 + k] = x[8 + k] + delta[6 + k];
    }
    __syncwarp();
}
// norm over the problem's parameter blocks, one component per lane (all lanes return the value)
__device__ __forceinline__ double norm14_warp(const double *v, int simple, int lane) {
    const bool mine = lane < 14 && (!simple || (lane >= 4 && lane < 8) || lane >= 11);
    return sqrt(warp_sum(mine ? v[lane] * v[lane] : 0.0));
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__device__ __forceinline__ void lm_step_device(const LmParams &P, int phase, LmScratch &S, IcpState *st, LmState *lm, int lane) {
    const double min_relative_decrease = 1e-3, function_tolerance = 1e-6, gradient_tolerance = 1e-10,
                 parameter_tolerance = 1e-8, min_radius = 1e-32, max_radius = 1e16, min_lm_diagonal = 1e-6,
                 max_lm_diagonal = 1e32;
    const int R = lm->num_residuals_global;
    // The scalar bookkeeping of TrustRegionMinimizer is a few dozen numbers: every loop over the 12 tangent directions /
    // 14 parameters runs one element per lane (reductions by shuffles), lane 0 keeps only the branchy decisions. (The
    // first cut ran them as serial loops on lane 0 against shared memory, several times slower.)

    // unpack the evaluation: U = J^T J, gu = J^T r, cost (+ regularisers at the evaluated point)
    for (int e = lane; e < 78; e += 32) {
        const int i = c_pair_i[e], j = c_pair_j[e];
        S.U[i][j] = S.acc[e];
        S.U[j][i] = S.acc[e];
    }
    if (lane < 12) S.gu[lane] = S.acc[78 + lane];
    __syncwarp();
    if (lane == 0) {
        S.cost = S.acc[kAccCost];
        if (!P.simple)   // AddConstraintsToCeresProblem only with CONTINUOUS_TIME (ct_icp.cpp:613)
            add_regularisers(&S.regs, R, phase == 0 ? lm->x : lm->cand, S.U, S.gu, S.cost);
        S.flag = 0;
    }
    __syncwarp();

    // adopt an evaluation as the current linearisation point (EvaluateGradientAndJacobian)
    auto adopt = [&](bool first) {
        for (int e = lane; e < 144; e += 32) lm->U[e / 12][e % 12] = S.U[e / 12][e % 12];
        if (lane < 12) {
            lm->gu[lane] = S.gu[lane];
            S.neg[lane] = -S.gu[lane];
            if (first) lm->scaling[lane] = 1.0 / (1.0 + sqrt(S.U[lane][lane]));   // jacobi_scaling, iteration 0 only
        }
        if (lane == 0) lm->x_cost = S.cost;
        __syncwarp();
        lm_plus_warp(lm->x, S.neg, S.proj, lane);
        const double gmax = warp_max(lane < 14 ? fabs(lm->x[lane] - S.proj[lane]) : 0.0);
        const double xn = norm14_warp(lm->x, P.simple, lane);
        if (lane == 0) {
            lm->gradient_max_norm = gmax;
            lm->x_norm = xn;
            lm->step_is_successful = 1;
        }
        __syncwarp();
    };

    if (phase == 0) {
        adopt(true);
    } else {
        // ComputeCandidatePointAndEvaluateCost happened in k_lm_eval; now the tolerance tests and the step decision
        const double dx = lane < 14 ? lm->x[lane] - lm->cand[lane] : 0.0;
        const double step_norm = sqrt(warp_sum(dx * dx));
        if (lane == 0) {
            const double candidate_cost = S.cost;
            const double cost_change = lm->x_cost - candidate_cost;
            if (step_norm <= parameter_tolerance * (lm->x_norm + parameter_tolerance)) {
                S.flag = 1;   // ParameterToleranceReached
            } else if (fabs(cost_change) <= function_tolerance * lm->x_cost) {
                S.flag = 1;   // FunctionToleranceReached
            } else {
                const double relative_decrease = cost_change / lm->model_cost_change;
                if (lm->trace_n < 256) {
                    double *tr = lm->trace[lm->trace_n++];
                    tr[0] = lm->x_cost; tr[1] = candidate_cost; tr[2] = lm->model_cost_change; tr[3] = relative_decrease;
                    tr[4] = lm->radius; tr[5] = relative_decrease > min_relative_decrease ? 1.0 : 0.0;
                    tr[6] = lm->x[0]; tr[7] = lm->x[1]; tr[8] = lm->x[2]; tr[9] = lm->x[3]; tr[10] = lm->x[11]; tr[11] = lm->x[12]; tr[12] = lm->x[13];
                }
                if (relative_decrease > min_relative_decrease) {
                    S.flag = 2;   // successful step
                    const double q3 = 2.0 * relative_decrease - 1.0;   // std::pow(·, 3) with an int exponent: repeated products
                    lm->radius = lm->radius / fmax(1.0 / 3.0, 1.0 - q3 * q3 * q3);
                    lm->radius = fmin(max_radius, lm->radius);
                    lm->decrease_factor = 2.0;
                    lm->reuse_diagonal = 0;
                } else {
                    S.flag = 3;   // rejected
                    lm->step_is_successful = 0;
                    lm->radius = lm->radius / lm->decrease_factor;
                    lm->decrease_factor *= 2.0;
                    lm->reuse_diagonal = 1;
                }
            }
        }
        __syncwarp();
        if (S.flag == 1) {
            if (lane == 0) lm->done = 1;
            return;
        }
        if (S.flag == 2) {
            if (lane < 14) lm->x[lane] = lm->cand[lane];
            __syncwarp();
            adopt(false);
        }
    }

    // main loop of TrustRegionMinimizer::Minimize until a candidate needs evaluating or the solve terminates
    for (int guard = 0; guard < 64; ++guard) {
        const bool improved = lm->step_is_successful && lm->x_cost < lm->minimum_cost;   // FinalizeIterationAndCheck…
        __syncwarp();
        if (improved && lane < 14) lm->best[lane] = lm->x[lane];
        if (lane == 0) {
            S.flag = 0;
            if (improved) lm->minimum_cost = lm->x_cost;
            if (lm->iteration >= P.ls_max_num_iters) S.flag = 1;
            else if (lm->step_is_successful && lm->gradient_max_norm <= gradient_tolerance) S.flag = 1;
            else if (lm->radius <= min_radius) S.flag = 1;
            else lm->iteration += 1;
        }
        __syncwarp();
        if (S.flag == 1) {
            if (lane == 0) lm->done = 1;
            return;
        }
        // LevenbergMarquardtStrategy::ComputeStep on the Jacobi-scaled system
        if (lane < 12 && !lm->reuse_diagonal) {
            const double sl = lm->scaling[lane];
            const double d = lm->U[lane][lane] * sl * sl;
            lm->diagonal[lane] = fmin(fmax(d, min_lm_diagonal), max_lm_diagonal);
        }
        __syncwarp();
        {
            const double inv_radius_num = lm->radius;
            for (int e = lane; e < 144; e += 32) {
                const int i = e / 12, j = e - 12 * i;
                double v = lm->U[i][j] * lm->scaling[i] * lm->scaling[j];
                if (i == j) v += lm->diagonal[i] / inv_radius_num;
                S.solve.A[i][j] = v;
            }
            if (lane < 12) S.solve.b[lane] = lm->gu[lane] * lm->scaling[lane];
        }
        __syncwarp();
        lm_solve12(S.solve, lane);   // (J'J + D^2) y = J'r
        if (lane < 12) S.step[lane] = -S.solve.x[lane];
        __syncwarp();
        // model_cost_change = -(J step)'(f + J step / 2) = -step'g - step'H step / 2   (scaled quantities)
        double sg_l = 0, shs_l = 0;
        bool finite_l = true;
        if (lane < 12) {   // row `lane` of H step, the twelve rows at once
            double hs = 0;
            for (int b = 0; b < 12; ++b) hs += lm->U[lane][b] * lm->scaling[lane] * lm->scaling[b] * S.step[b];
            sg_l = S.step[lane] * lm->gu[lane] * lm->scaling[lane];
            shs_l = S.step[lane] * hs;
            finite_l = isfinite(S.step[lane]);
            S.delta[lane] = S.step[lane] * lm->scaling[lane];
        }
        const double sg = warp_sum(sg_l), shs = warp_sum(shs_l);
        const bool finite = __all_sync(0xffffffffu, finite_l);
        const double mcc = -sg - 0.5 * shs;
        const bool valid_step = finite && mcc > 0.0;
        if (lane == 0) {
            lm->reuse_diagonal = 1;
            lm->model_cost_change = mcc;
            if (!valid_step) {   // HandleInvalidStep
                lm->num_invalid += 1;
                if (lm->num_invalid >= 5) {
                    lm->usable = 0;
                    S.flag = 1;
                } else {
                    lm->radius *= 0.5;
                    lm->reuse_diagonal = 1;
                    lm->step_is_successful = 0;
                    S.flag = 4;   // loop again
                }
            } else {
                lm->num_invalid = 0;
            }
        }
        __syncwarp();
        if (valid_step) lm_plus_warp(lm->x, S.delta, lm->cand, lane);
        if (S.flag == 1) {
            if (lane == 0) lm->done = 1;
            return;
        }
        if (S.flag == 4) continue;
        return;   // candidate ready → k_lm_eval(which = 1)
    }
}

template <bool kPeers>
__global__ void __launch_bounds__(128)
k_lm_step(LmParams P, int phase, const double *__restrict__ partials, int nblocks, IcpState *st, LmState *lm,
          PeerLinks links) {
    __shared__ LmScratch S;
    __shared__ double s_part[4][kAcc];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (st->done || lm->done) return;
    {   // deterministic reduction of the evaluation partials
        double a0 = 0, a1 = 0, a2 = 0;
        for (int b = w; b < nblocks; b += 4) {
            const double *row = partials + (size_t) b * kAcc;
            a0 += row[lane];
            a1 += row[lane + 32];
            a2 += row[lane + 64];
        }
        s_part[w][lane] = a0;
        s_part[w][lane + 32] = a1;
        s_part[w][lane + 64] = a2;
        __syncthreads();
        if (threadIdx.x < kAcc) S.acc[threadIdx.x] = s_part[0][threadIdx.x] + s_part[1][threadIdx.x] + s_part[2][threadIdx.x] + s_part[3][threadIdx.x];
        __syncthreads();
    }
    if (kPeers) {
        __shared__ unsigned int s_half[kMaxPeers * kPeerWords];
        __shared__ int s_peer_ok;
        const unsigned int seq = *links.seq + 1;
        const bool ok = peer_allreduce(links, seq, S.acc, s_half, &s_peer_ok);   // Σ over ranks, in rank order
        if (threadIdx.x == 0) {
            *links.seq = seq;
            if (!ok) {   // a peer never answered: give up instead of hanging the device
                st->failed = 3;
                st->done = 1;
            }
        }
        if (!ok) return;
    }
    if (w != 0) return;
    lm_load_regs(S.regs, st, lane);
    lm_step_device(P, phase, S, st, lm, lane);
}

// end of one ICP iteration (ct_icp.cpp:636-672): write the pose pair back and test the stop criterion
// one thread
__device__ __forceinline__ void lm_finish_device(const LmParams &P, IcpState *st, LmState *lm, int outer_index) {
    if (!lm->usable) {   // reference: throw std::runtime_error("Error During Optimization") (:639-642)
        st->failed = 2;
        st->done = 1;
        return;
    }
    const Q4 qb = qnormalized(Q4{lm->best[0], lm->best[1], lm->best[2], lm->best[3]});
    const Q4 qe = qnormalized(Q4{lm->best[4], lm->best[5], lm->best[6], lm->best[7]});
    st->qb[0] = qb.x; st->qb[1] = qb.y; st->qb[2] = qb.z; st->qb[3] = qb.w;
    st->qe[0] = qe.x; st->qe[1] = qe.y; st->qe[2] = qe.z; st->qe[3] = qe.w;
    for (int d = 0; d < 3; ++d) {
        st->tb[d] = lm->best[8 + d];
        st->te[d] = lm->best[11 + d];
    }
    const SlerpConsts sc = slerp_consts(qb, qe);
    st->slerp_theta = sc.theta;
    st->slerp_inv_sin = sc.inv_sin;
    st->slerp_linear = sc.linear;
    st->slerp_negate = sc.negate;
    double dtb = 0, dte = 0;
    for (int d = 0; d < 3; ++d) {
        dtb += (lm->prev_tb[d] - st->tb[d]) * (lm->prev_tb[d] - st->tb[d]);
        dte += (lm->prev_te[d] - st->te[d]) * (lm->prev_te[d] - st->te[d]);
    }
    const double diff_trans = sqrt(dtb) + sqrt(dte);
    const double diff_rot = angular_distance_deg(qb, Q4{lm->prev_qb[0], lm->prev_qb[1], lm->prev_qb[2], lm->prev_qb[3]}) +
                            angular_distance_deg(qe, Q4{lm->prev_qe[0], lm->prev_qe[1], lm->prev_qe[2], lm->prev_qe[3]});
    for (int d = 0; d < 4; ++d) { lm->prev_qb[d] = st->qb[d]; lm->prev_qe[d] = st->qe[d]; }
    for (int d = 0; d < 3; ++d) { lm->prev_tb[d] = st->tb[d]; lm->prev_te[d] = st->te[d]; }
    st->iter = outer_index + 1;
    if (diff_rot < P.threshold_orientation_norm && diff_trans < P.threshold_translation_norm) {
        st->iter = outer_index;   // the reference's loop index at `break` (:668-672)
        st->done = 1;
    }
}

__global__ void k_lm_finish(LmParams P, IcpState *st, LmState *lm, int outer_index) {
    if (threadIdx.x != 0 || st->done) return;
    lm_finish_device(P, st, lm, outer_index);
}

// one thread
__device__ __forceinline__ void lm_begin_device(IcpState *st, LmState *lm, unsigned long long *stats) {
    for (int d = 0; d < 4; ++d) { lm->prev_qb[d] = st->qb[d]; lm->prev_qe[d] = st->qe[d]; }
    for (int d = 0; d < 3; ++d) { lm->prev_tb[d] = st->tb[d]; lm->prev_te[d] = st->te[d]; }
    lm->done = 0;
    lm->usable = 1;
    lm->trace_n = 0;
    stats[0] = 0;
    stats[1] = 0;
}
__global__ void k_lm_begin(IcpState *st, LmState *lm, unsigned long long *stats) {
    if (threadIdx.x != 0) return;
    lm_begin_device(st, lm, stats);
}

// ---- persistent variant: the WHOLE CERES / ROBUST registration of a frame in one cooperative launch -------------------
// The reference's DoRegisterCeres / DoRegisterRobust loop (ct_icp.cpp:549-672, 1229-1336) — per ICP iteration: residual
// assembly, GetProblem, ceres::Solve (one evaluation + up to ls_max_num_iters candidate evaluations, each followed by a
// trust-region step), stop test — used to be ~15 launches per ICP iteration. Here CTA 0 is the SOLVER CTA: it runs
// GetProblem and the minimizer with the whole LM state in its shared memory (the serial trust-region logic no longer pays
// global-memory latency on every access) and publishes the candidate point; CTAs 1..G assemble the residual blocks
// (gather + selection, tiled) and evaluate the residuals / Jacobians (half a warp per block). Grid-wide barriers separate
// the phases: 2 per ICP iteration + 2 per evaluation. Sharded (kPeers): the per-rank valid counts and every evaluation's
// accumulator are exchanged by the solver CTA over the NVLink peer mailboxes, inside the loop.
// kMode: 0 = CERES with the nearest-neighbor strategy, 1 = CERES with the distance-based strategy, 2 = ROBUST.
constexpr int kLmPWarps = 16;
struct LmSolverShared {
    LmScratch S;
    double part[kLmPWarps][kAcc];
    LmSelectScratch sel;
    unsigned int half[kMaxPeers * kPeerWords];
    LmState lm;
};
struct LmEvalShared {
    double u[kLmPWarps * 2][16];
    double acc[kLmPWarps * 2][kAcc];
};
struct __align__(16) LmPShared {
    union {
        LmTile tile[kLmPWarps];   // workers, assembly phase
        LmEvalShared eval;        // workers, evaluation phase
        LmSolverShared solver;    // CTA 0
    };
    int stencil[kMaxStencil];
    int flag;
    int next;   // tile counter of the residual assembly (lm_grab_tile)
};
static_assert(sizeof(LmPShared) <= 227 * 1024, "k_lm_persistent: dynamic shared memory of one CTA (sm_90: 227 KB)");
extern __shared__ __align__(16) unsigned char lm_smem_raw[];

// what the worker CTAs read of the LM state: the point to evaluate, the problem size, the stop flag
__device__ __forceinline__ void lm_publish(LmState *dst, const LmState *src, int tid) {
    if (tid < 14) {
        __stcg(&dst->x[tid], src->x[tid]);
        __stcg(&dst->cand[tid], src->cand[tid]);
    }
    if (tid == 0) {
        __stcg(&dst->num_residuals, src->num_residuals);
        __stcg(&dst->done, src->done);
    }
}

// One registration of a grouped k_lm_persistent launch (LmGroups): everything a solo launch takes as kernel parameters.
// Groups may search different maps with different options and buffers (the odometry's batch: one handle per group).
struct LmGroup {
    GatherConfig G;              // map level and search of the default radius
    LmParams P;                  // options; P.kp_lo: the group's residual plane
    const float4 *keypoints;
    const int *num_keypoints;    // device count
    IcpState *st;
    ResidualBlock *blocks;       // the group's residual blocks, sel_idx and (ROBUST) classes
    int *sel_idx;
    unsigned char *classes;
    const DistanceStrategy *D;   // mode 1
};

// The groups of one grouped k_lm_persistent launch (k_lm_persistent<mode, false, true>). Group g owns the CTAs
// [first_cta[g], first_cta[g + 1]) of the grid — the first is g's solver CTA, the others its workers — the registration
// table[g], and in the launch-wide area the LmState at kLmStateStride · g, its stats line, the partial rows
// [first_cta[g] - g, first_cta[g + 1] - g - 1) and its barrier words. `table` (device) = LmGroup[B] | first_cta[0..B]
// (IcpSolver::EnqueueCeresGroups).
struct LmGroups {
    const LmGroup *table;
    int num_groups;
    unsigned int *barrier;   // kLmBarrierWords per group: arrival counter at [0], abort word at [32]; zeroed before each launch
};
// dynamic shared memory of the grouped instantiations: the solo kernel's, then the CTA's entry of the table
constexpr size_t kLmGroupedShared = sizeof(LmPShared) + sizeof(LmGroup);
static_assert(kLmGroupedShared <= 227 * 1024, "k_lm_persistent<mode, false, true>: dynamic shared memory of one CTA");
static_assert(sizeof(LmGroup) % sizeof(int) == 0, "the CTAs copy their entry word by word");
constexpr int kLmBarrierWords = 64;                                        // two 128-byte lines per group
constexpr size_t kLmStateStride = (sizeof(LmState) + 127) / 128 * 128;     // LmStates of the groups on separate lines
constexpr int kLmStatsStride = 16;                                         // one 128-byte line of stats per group

__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int *p) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// The grid barrier of cooperative groups, scoped to one group of CTAs: every CTA of the group arrives once per barrier, so
// the group's barrier k completes when its counter reaches `target` = k · group_ctas. The wait is bounded: a CTA that has
// waited kLoopSyncTimeout cycles sets the group's abort word; a waiter that finds it set leaves too. Returns false
// (uniform over the CTA) when the group was aborted. Groups share nothing, so a stalled group never holds up another.
// Called by all threads of the CTA.
__device__ __forceinline__ bool lm_group_barrier(unsigned int *bar, unsigned int target) {
    __syncthreads();
    int ok = 1;
    if (threadIdx.x == 0) {
        unsigned int *count = bar, *abort = bar + 32;
        __threadfence();
        atomicAdd(count, 1u);
        const long long t0 = clock64();
        while (ld_acquire_u32(count) < target) {
            if (ld_acquire_u32(abort)) {
                ok = 0;
                break;
            }
            if (clock64() - t0 > kLoopSyncTimeout) {
                atomicExch(abort, 1u);
                ok = 0;
                break;
            }
        }
    }
    return __syncthreads_and(ok) != 0;
}

// The registration of one group: `cta` is this CTA's index in it, `group_ctas` its size, and every pointer is the group's
// own. Solo (kGrouped false): the whole grid, separated by grid-wide barriers. Grouped: group barriers (lm_group_barrier at
// `bar`); when one times out every CTA of the group leaves the loop and the solver CTA marks the state failed = 2.
template <int kMode, bool kPeers, bool kGrouped>
__device__ __forceinline__ void lm_persistent_body(const GatherConfig &G0, const LmParams &P, const float4 *__restrict__ keypoints,
                                                   const int *__restrict__ d_num_keypoints, IcpState *st, LmState *lm_g,
                                                   ResidualBlock *__restrict__ blocks, int *__restrict__ sel_idx,
                                                   unsigned char *__restrict__ classes, unsigned long long *stats,
                                                   const DistanceStrategy *__restrict__ D, double *__restrict__ partials,
                                                   PeerLinks links, int cta, int group_ctas, unsigned int *bar) {
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    unsigned int barriers = 0;   // grouped: barriers taken so far
    const auto sync = [&]() -> bool {
        if constexpr (kGrouped) {
            return lm_group_barrier(bar, ++barriers * (unsigned int) group_ctas);
        } else {
            grid.sync();
            return true;
        }
    };
    bool live = true;   // grouped: false once the group has been aborted
    LmPShared &sh = *reinterpret_cast<LmPShared *>(lm_smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const bool solver = cta == 0;
    const int workers = group_ctas - 1, wi = cta - 1;
    const int *stencil = kMode == 1 ? nullptr : stencil_table_fill(sh.stencil, G0.r);
    LmState *lm = &sh.solver.lm;   // the solver CTA's working copy (shared memory); lm_g is what the workers see
    unsigned int peer_seq = 0;
    if (solver) {
        if (kPeers) peer_seq = *links.seq;
        if (w == 1) lm_load_regs(sh.solver.S.regs, st, lane);
        if (tid == 0) lm_begin_device(st, lm, stats);
        __syncthreads();
        lm_publish(lm_g, lm, tid);
        __threadfence();
    }
    live = sync();
    const int K = *d_num_keypoints;
    CT_STAMP(long long t_mark = clock64(); const long long t_loop = t_mark;)
    CT_STAMP(if (solver && tid < 8) lm->dbg_cycles[tid] = 0;)
#define LM_STAMP(slot) CT_STAMP(if (solver && tid == 0) { const long long now = clock64(); lm->dbg_cycles[slot] += (unsigned long long) (now - t_mark); t_mark = now; })

    for (int it = 0; live && it < P.num_iters_icp; ++it) {
        if (__ldcg(&st->done)) break;   // uniform (over the group): written before a barrier
        // ---- residual assembly (workers)
        if (!solver) {
            // (every warp of this CTA left the previous assembly before the grid barriers in between)
            if (tid == 0) sh.next = 0;
            __syncthreads();
            if (kMode == 2)
                rb_gather_tiles<kGrouped>(G0, P, stencil, keypoints, K, st, blocks, classes, stats, sh.tile[w], wi, workers, kLmPWarps, &sh.next, lane);
            else if (kMode == 1)
                lm_gather_tiles<true, kGrouped>(G0, P, stencil, keypoints, K, st, blocks, stats, D, sh.tile[w], wi, workers, kLmPWarps, &sh.next, lane);
            else
                lm_gather_tiles<false, kGrouped>(G0, P, stencil, keypoints, K, st, blocks, stats, D, sh.tile[w], wi, workers, kLmPWarps, &sh.next, lane);
        }
        if (!sync()) {
            live = false;
            break;
        }
        LM_STAMP(1)
        // ---- GetProblem (solver): the first max_num_residuals valid blocks in keypoint order, seeds the minimizer
        if (solver) {
            double *counts = sh.solver.part[0];
            if (kPeers) {   // all-gather of the per-rank valid counts (as a sum of one-hot vectors)
                if (tid < kAcc) counts[tid] = 0.0;
                __syncthreads();
                lm_select_device(P, 1, K, blocks, sel_idx, st, lm, stats, counts, sh.solver.sel);
                const bool ok = peer_allreduce(links, ++peer_seq, counts, sh.solver.half, &sh.flag);
                if (!ok && tid == 0) {
                    st->failed = 3;
                    st->done = 1;
                }
                __syncthreads();
            }
            if (!__ldcg(&st->done)) lm_select_device(P, 0, K, blocks, sel_idx, st, lm, stats, counts, sh.solver.sel);
            __syncthreads();
            lm_publish(lm_g, lm, tid);
            __threadfence();
        }
        LM_STAMP(2)
        if (!sync()) {
            live = false;
            break;
        }
        LM_STAMP(6)
        // ---- ceres::Solve: evaluation 0 at x, then one evaluation per candidate
        for (int ev = 0; ev <= P.ls_max_num_iters; ++ev) {
            if (__ldcg(&st->done) || __ldcg(&lm_g->done)) break;   // uniform
            const int phase = ev > 0 ? 1 : 0;
            if (!solver) {
                const int hw = w * 2 + (lane >> 4);
                lm_eval_device<kLmPWarps * 2, kGrouped>(P, phase, blocks, sel_idx, st, lm_g, sh.eval.u, sh.eval.acc,
                                              hw * workers + wi, workers * kLmPWarps * 2, partials + (size_t) wi * kAcc);
            }
            if (!sync()) {
                live = false;
                break;
            }
            LM_STAMP(3)
            CT_STAMP(if (solver && tid == 0) lm->dbg_cycles[7] += 1;)
            if (solver) {
                // deterministic reduction of the workers' rows: warp g sums the rows b = g (mod warps), all its loads in
                // flight before the first add; then the per-warp sums in fixed order
                {
                    constexpr int kInFlight = 10;
                    double a0 = 0, a1 = 0, a2 = 0;
                    for (int b0 = w; b0 < workers; b0 += kLmPWarps * kInFlight) {
                        double v0[kInFlight], v1[kInFlight], v2[kInFlight];
#pragma unroll
                        for (int u = 0; u < kInFlight; ++u) {
                            const int b = b0 + u * kLmPWarps;
                            v0[u] = v1[u] = v2[u] = 0.0;
                            if (b < workers) {
                                const double *row = partials + (size_t) b * kAcc;
                                v0[u] = __ldcg(row + lane);
                                v1[u] = __ldcg(row + lane + 32);
                                v2[u] = __ldcg(row + lane + 64);
                            }
                        }
#pragma unroll
                        for (int u = 0; u < kInFlight; ++u)
                            if (b0 + u * kLmPWarps < workers) {
                                a0 += v0[u];
                                a1 += v1[u];
                                a2 += v2[u];
                            }
                    }
                    sh.solver.part[w][lane] = a0;
                    sh.solver.part[w][lane + 32] = a1;
                    sh.solver.part[w][lane + 64] = a2;
                    __syncthreads();
                    if (tid < kAcc) {
                        double sum = 0;
#pragma unroll
                        for (int ww = 0; ww < kLmPWarps; ++ww) sum += sh.solver.part[ww][tid];
                        sh.solver.S.acc[tid] = sum;
                    }
                    __syncthreads();
                }
                LM_STAMP(4)
                bool ok = true;
                if (kPeers) ok = peer_allreduce(links, ++peer_seq, sh.solver.S.acc, sh.solver.half, &sh.flag);
                if (w == 0) {
                    if (!ok) {
                        if (lane == 0) {   // a peer never answered: give up instead of hanging the device
                            st->failed = 3;
                            st->done = 1;
                        }
                    } else {
                        lm_step_device(P, phase, sh.solver.S, st, lm, lane);
                        __syncwarp();
                        // the solve has terminated: pose write-back + stop test of the ICP loop (ct_icp.cpp:636-672)
                        if (lane == 0 && lm->done && !st->done) lm_finish_device(P, st, lm, it);
                    }
                }
                __syncthreads();
                lm_publish(lm_g, lm, tid);
                __threadfence();
            }
            LM_STAMP(5)
            if (!sync()) {
                live = false;
                break;
            }
            LM_STAMP(6)
        }
        if (!live) break;
    }
    CT_STAMP(if (solver && tid == 0) lm->dbg_cycles[0] = (unsigned long long) (clock64() - t_loop);)
#undef LM_STAMP
    if (solver) {
        if (kPeers && tid == 0) *links.seq = peer_seq;
        if (kGrouped && !live && tid == 0) {   // a CTA of the group never arrived: the problem fails, the others go on
            st->failed = 2;
            st->done = 1;
        }
        // the whole state (incl. the debug trace) for the host
        __syncthreads();
        const int words = (int) (sizeof(LmState) / sizeof(int));
        const int *src = reinterpret_cast<const int *>(lm);
        int *dst = reinterpret_cast<int *>(lm_g);
        for (int i = tid; i < words; i += blockDim.x) dst[i] = src[i];
    }
}

// kGrouped: one launch runs the groups of `groups` (EnqueueCeresGroups), each CTA with its group's entry copied to shared
// memory behind LmPShared (kLmGroupedShared), and the parameters G0 … D are not read (lm_g, stats and partials are the
// launch-wide areas); otherwise the grid is one registration and `groups` is not read.
template <int kMode, bool kPeers, bool kGrouped = false>
__global__ void __launch_bounds__(kLmPWarps * 32, 1)
k_lm_persistent(GatherConfig G0, LmParams P, const float4 *__restrict__ keypoints, const int *__restrict__ d_num_keypoints,
                IcpState *st, LmState *lm_g, ResidualBlock *__restrict__ blocks, int *__restrict__ sel_idx,
                unsigned char *__restrict__ classes, unsigned long long *stats, const DistanceStrategy *__restrict__ D,
                double *__restrict__ partials, PeerLinks links, LmGroups groups) {
    if constexpr (kGrouped) {
        static_assert(!kPeers, "a batched launch is not sharded");
        const int *first_cta = reinterpret_cast<const int *>(groups.table + groups.num_groups);
        int g = 0;
        while (first_cta[g + 1] <= (int) blockIdx.x) ++g;
        LmGroup &e = *reinterpret_cast<LmGroup *>(lm_smem_raw + sizeof(LmPShared));
        {
            const int *src = reinterpret_cast<const int *>(groups.table + g);
            int *dst = reinterpret_cast<int *>(&e);
            for (int i = threadIdx.x; i < (int) (sizeof(LmGroup) / sizeof(int)); i += blockDim.x) dst[i] = src[i];
        }
        __syncthreads();
        lm_persistent_body<kMode, false, true>(
            e.G, e.P, e.keypoints, e.num_keypoints, e.st,
            reinterpret_cast<LmState *>(reinterpret_cast<char *>(lm_g) + kLmStateStride * g), e.blocks, e.sel_idx, e.classes,
            stats + (size_t) kLmStatsStride * g, e.D, partials + (size_t) (first_cta[g] - g) * kAcc, links,
            (int) blockIdx.x - first_cta[g], first_cta[g + 1] - first_cta[g], groups.barrier + (size_t) kLmBarrierWords * g);
    } else {
        lm_persistent_body<kMode, kPeers, false>(G0, P, keypoints, d_num_keypoints, st, lm_g, blocks, sel_idx, classes, stats,
                                                 D, partials, links, (int) blockIdx.x, (int) gridDim.x, nullptr);
    }
}

// ---------------------------------------------------------------------------------------------------------------
void IcpSolver::EnsureLmBuffers(size_t k_upper) {
    d_lm_state_.reserve(1, stream_);
    d_lm_stats_.reserve(2, stream_);
    d_lm_classes_.reserve(k_upper, stream_);
    d_lm_blocks_.reserve(k_upper, stream_);
    d_lm_sel_.reserve(k_upper, stream_);
}
void IcpSolver::PreloadLmKernels() {
    cudaFuncAttributes a;
    cudaFuncGetAttributes(&a, k_lm_step<true>);
    cudaFuncGetAttributes(&a, k_lm_step<false>);
    cudaFuncGetAttributes(&a, k_lm_eval);
    cudaFuncGetAttributes(&a, k_lm_gather<false>);
    cudaFuncGetAttributes(&a, k_lm_gather<true>);
    cudaFuncGetAttributes(&a, k_rb_gather);
    cudaFuncGetAttributes(&a, k_lm_select);
}

// k_lm_persistent<mode, peers, grouped>; mode 0 = CERES nearest neighbor, 1 = CERES distance-based, 2 = ROBUST
static void *LmPersistentKernel(int mode, bool peers, bool grouped) {
    if (grouped) return mode == 0 ? (void *) k_lm_persistent<0, false, true>
                      : mode == 1 ? (void *) k_lm_persistent<1, false, true>
                                  : (void *) k_lm_persistent<2, false, true>;
    switch (mode * 2 + (peers ? 1 : 0)) {
        case 0: return (void *) k_lm_persistent<0, false>;
        case 1: return (void *) k_lm_persistent<0, true>;
        case 2: return (void *) k_lm_persistent<1, false>;
        case 3: return (void *) k_lm_persistent<1, true>;
        case 4: return (void *) k_lm_persistent<2, false>;
        default: return (void *) k_lm_persistent<2, true>;
    }
}
int IcpSolver::LmCoresident(int variant, void *kernel, size_t smem) {
    int &coresident = lm_coresident_[variant];
    if (coresident == 0) {
        CT_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
        int per_sm = 0;
        CT_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kLmPWarps * 32, smem));
        coresident = std::max(1, per_sm * num_sms_);
    }
    return coresident;
}

// the DistanceBasedStrategy's parameters and every map level → d_lm_strategy_ when solver CERES uses that strategy
// (ct_icp.cpp:571; ROBUST does not consult the strategy, :1235). Options checked by CheckCeresOptions. Returns whether it does.
bool IcpSolver::UploadLmStrategy(const DeviceMap &map, const cticp_icp_options &opt, const cticp_strategy_options &strategy) {
    if (opt.solver == CTICP_SOLVER_ROBUST || strategy.type != CTICP_STRATEGY_DISTANCE_BASED) return false;
    DistanceStrategy D{};
    D.num_levels = map.NumLevels();
    D.filter = map.Options().select_valid_normals_direction ? 1 : 0;
    D.radius_min = strategy.radius_min;
    D.radius_max = strategy.radius_max;
    D.exponent = strategy.exponent;
    for (int i = 0; i < D.num_levels; ++i) D.levels[i] = map.Level(i);
    d_lm_strategy_.reserve(1, stream_);
    CT_CUDA_CHECK(cudaMemcpyAsync(d_lm_strategy_.data(), &D, sizeof(D), cudaMemcpyHostToDevice, stream_));
    CT_CUDA_CHECK(cudaStreamSynchronize(stream_));   // D lives on this stack frame
    return true;
}

// the parameters of the LM kernels for checked options (CheckCeresOptions)
static LmParams MakeLmParams(const DeviceMap &map, const cticp_icp_options &opt, const cticp_strategy_options &strategy,
                             const float4 *kp_lo, int shard_rank, int shard_world) {
    const bool robust = opt.solver == CTICP_SOLVER_ROBUST;
    const double sum = std::abs(opt.weight_alpha) + std::abs(opt.weight_neighborhood);
    LmParams P{};
    P.ncn = robust ? 1 : opt.num_closest_neighbors;
    map.SearchParams(map.Options().default_radius, &P.level, &P.r);
    P.radius = map.Options().default_radius;
    P.bucket_scale = (double) kSelBuckets / (P.radius * P.radius);
    P.kp_lo = kp_lo;
    // neighbor count: the strategy's for CERES (neighborhood_strategy.h:81), the ICP options' for ROBUST (:1235)
    P.kmax = robust ? opt.max_number_neighbors : strategy.max_num_neighbors;
    P.kmin = opt.min_number_neighbors;            // ct_icp.cpp:574
    P.lambda_weight = std::abs(opt.weight_alpha) / sum;
    P.lambda_neighborhood = std::abs(opt.weight_neighborhood) / sum;
    P.power_planarity = opt.power_planarity;
    P.max_dist_to_plane = opt.max_dist_to_plane_ct_icp;
    P.max_num_residuals = opt.max_num_residuals;
    P.min_number_neighbors = opt.min_number_neighbors;
    P.num_iters_icp = opt.num_iters_icp;
    P.threshold_orientation_norm = opt.threshold_orientation_norm;
    P.threshold_translation_norm = opt.threshold_translation_norm;
    P.loss = make_loss(opt.loss_function, opt.ls_sigma, opt.ls_tolerant_min_threshold);
    P.ls_max_num_iters = opt.ls_max_num_iters;
    P.shard_rank = shard_rank;
    P.shard_world = shard_world;
    P.robust = robust ? 1 : 0;
    // solver ROBUST ignores the parametrization (DoRegisterRobust is CONTINUOUS_TIME only, ct_icp.cpp:1180-1370)
    P.simple = (!robust && opt.parametrization == CTICP_PARAM_SIMPLE) ? 1 : 0;
    P.distortion = opt.point_to_plane_with_distortion ? 1 : 0;
    P.use_lines = opt.use_lines;
    P.use_barycenter = opt.use_barycenter;
    P.threshold_linearity = opt.threshold_linearity;
    P.threshold_planarity = opt.threshold_planarity;
    P.outlier_distance = opt.outlier_distance;
    P.weight_neighborhood = opt.weight_neighborhood;
    return P;
}
static GatherConfig LmGatherConfig(const DeviceMap &map, const LmParams &P) {
    GatherConfig G;
    G.L = map.Level(P.level);
    G.r = P.r;
    G.radius2 = P.radius * P.radius;
    G.kmax = P.kmax;
    return G;
}

void IcpSolver::CheckCeresOptions(const DeviceMap &map, const cticp_icp_options &opt,
                                  const cticp_strategy_options &strategy) const {
    const bool robust = opt.solver == CTICP_SOLVER_ROBUST;
    if (!robust && opt.distance != CTICP_DIST_POINT_TO_PLANE)
        throw UnsupportedError("solver CERES: only POINT_TO_PLANE is built (SURVEY §8)");
    // ct_icp.cpp:593-601 indexes neighborhood.points[i] for i < num_closest_neighbors: defined only while a described
    // neighborhood has at least that many points (>= max(min_number_neighbors, 5))
    const int ncn = robust ? 1 : opt.num_closest_neighbors;
    if (ncn < 1 || ncn > kMaxNcn || ncn > std::max(opt.min_number_neighbors, 5))
        throw UnsupportedError("solver CERES: num_closest_neighbors must be in [1, min(4, min_number_neighbors)]");
    if (robust && opt.min_number_neighbors < 5)
        throw UnsupportedError("solver ROBUST: min_number_neighbors < 5 (neighborhoods the reference cannot describe, "
                               "neighborhood.h:227, and then reads stale) is not built");
    // neighbor count: the strategy's for CERES (neighborhood_strategy.h:81), the ICP options' for ROBUST (:1235)
    const int kmax = robust ? opt.max_number_neighbors : strategy.max_num_neighbors;
    if (kmax > 32 || kmax < 1) throw std::invalid_argument("max_num_neighbors must be in [1, 32]");
    const double sum = std::abs(opt.weight_alpha) + std::abs(opt.weight_neighborhood);
    if (!(sum > 0.0)) throw std::invalid_argument("weight_alpha + weight_neighborhood <= 0");
    // solver CERES consults the neighborhood strategy (ct_icp.cpp:571); ROBUST does not (:1235)
    if (!robust && strategy.type == CTICP_STRATEGY_DISTANCE_BASED) {
        if (!(strategy.radius_max > 0.0)) throw std::invalid_argument("DISTANCE_BASED_STRATEGY: radius_max must be > 0");
        if (map.Options().select_valid_normals_direction && !map.HasNormals())
            throw std::invalid_argument("DISTANCE_BASED_STRATEGY with select_valid_normals_direction needs a map that keeps normals");
    } else if (!robust && strategy.type != CTICP_STRATEGY_NEAREST_NEIGHBOR) {
        throw std::invalid_argument("unknown neighborhood strategy type");
    }
}


void IcpSolver::EnqueueCeres(const DeviceMap &map, const cticp_icp_options &opt, const cticp_strategy_options &strategy,
                             const float4 *d_keypoints, const int *d_num_keypoints, size_t k_hint, size_t k_capacity,
                             IcpState *d_state, int shard_rank, int shard_world, void *nccl_comm) {
    CheckCeresOptions(map, opt, strategy);
    const bool robust = opt.solver == CTICP_SOLVER_ROBUST;
    const int ncn = robust ? 1 : opt.num_closest_neighbors;
    const bool sharded = nccl_comm != nullptr && shard_world > 1;
    EnsureLmBuffers(k_capacity * (size_t) ncn);
    LmParams P = MakeLmParams(map, opt, strategy, kp_lo_, sharded ? shard_rank : 0, sharded ? shard_world : 1);
    if (sharded && shard_world > kAcc) throw std::invalid_argument("sharding: world size above 96");
    const GatherConfig G = LmGatherConfig(map, P);

    auto *lm = d_lm_state_.data();
    auto *blocks_buf = d_lm_blocks_.data();
    auto *stats = d_lm_stats_.data();
    const int gather_blocks = (int) std::max<size_t>(1, std::min<size_t>((k_hint + kLmWarps - 1) / kLmWarps, (size_t) num_sms_ * 8));
    const size_t r_hint = opt.max_num_residuals > 0 ? std::min<size_t>(k_hint, (size_t) opt.max_num_residuals) : k_hint;
    const int eval_blocks = (int) std::max<size_t>(1, std::min<size_t>((r_hint + kLmWarps * 2 - 1) / (kLmWarps * 2), (size_t) num_sms_ * 4));
    EnsurePartials(eval_blocks);

    const bool distance_based = UploadLmStrategy(map, opt, strategy);
    auto *classes = d_lm_classes_.data();
    if (robust) CT_CUDA_CHECK(cudaMemsetAsync(classes, 0, k_capacity, stream_));   // NEIGHBORHOOD_TYPE::NONE

    if (use_persistent_ && (!sharded || peers_ready_)) {
        // one cooperative launch for the whole registration (k_lm_persistent); the grid must be co-resident
        const int mode = robust ? 2 : (distance_based ? 1 : 0);
        const bool peers = sharded;
        void *kernel = LmPersistentKernel(mode, peers, false);
        const int coresident = LmCoresident(mode * 2 + (peers ? 1 : 0), kernel, sizeof(LmPShared));
        const size_t k_share = (k_hint + (size_t) P.shard_world - 1) / (size_t) P.shard_world + 16;
        int grid = (int) std::min<size_t>((size_t) coresident, 1 + std::max<size_t>(1, (k_share + kp_per_cta_ - 1) / kp_per_cta_));
        grid = std::max(grid, 2);
        EnsurePartials(grid);
        const float4 *kp = d_keypoints;
        const int *nk = d_num_keypoints;
        int *sel = d_lm_sel_.data();
        const DistanceStrategy *dstrat = d_lm_strategy_.data();
        double *parts = d_partials_.data();
        PeerLinks links = peers ? PeerLinksOf(links_host_) : PeerLinks{};
        LmGroups groups{};
        GatherConfig g = G;
        void *args[] = {&g, &P, &kp, &nk, &d_state, &lm, &blocks_buf, &sel, &classes, &stats, &dstrat, &parts, &links, &groups};
        const bool timed = time_gather_ && ev_used_ < kMaxEvents;
        if (timed) cudaEventRecord(ev_begin_[ev_used_].get(), stream_);
        CT_CUDA_CHECK(cudaLaunchCooperativeKernel(kernel, dim3(grid), dim3(kLmPWarps * 32), args, sizeof(LmPShared), stream_));
        if (timed) cudaEventRecord(ev_end_[ev_used_++].get(), stream_);
        gather_launches_ += 1;
        launches_ += 1;
        DebugLmTrace(lm);
        return;
    }

    k_lm_begin<<<1, 32, 0, stream_>>>(d_state, lm, stats);
    launches_ += 1;
    for (int it = 0; it < opt.num_iters_icp; ++it) {
        const bool timed = time_gather_ && ev_used_ < kMaxEvents;
        if (timed) cudaEventRecord(ev_begin_[ev_used_].get(), stream_);
        if (robust)
            k_rb_gather<<<gather_blocks, kLmWarps * 32, 0, stream_>>>(G, P, d_keypoints, d_num_keypoints, d_state, blocks_buf,
                                                                     classes, stats);
        else if (distance_based)
            k_lm_gather<true><<<gather_blocks, kLmWarps * 32, 0, stream_>>>(G, P, d_keypoints, d_num_keypoints, d_state, blocks_buf,
                                                                           stats, d_lm_strategy_.data());
        else
            k_lm_gather<false><<<gather_blocks, kLmWarps * 32, 0, stream_>>>(G, P, d_keypoints, d_num_keypoints, d_state, blocks_buf,
                                                                            stats, nullptr);
        if (timed) cudaEventRecord(ev_end_[ev_used_++].get(), stream_);
        ++gather_launches_;
        // One evaluation + minimizer step. Sharded: every rank evaluates its share of the residual blocks, the 96-double
        // accumulators are summed over the ranks (ncclAllReduce, bit-identical result everywhere) and every rank takes
        // the same step — the exchange of SURVEY §8e, once per LM evaluation.
        auto eval_and_step = [&](int phase) {
            k_lm_eval<<<eval_blocks, kLmWarps * 32, 0, stream_>>>(P, phase, blocks_buf, d_lm_sel_.data(), d_state, lm, d_partials_.data());
            if (sharded && peers_ready_) {   // exchange inside the step kernel (NVLink peer mailboxes)
                k_lm_step<true><<<1, 128, 0, stream_>>>(P, phase, d_partials_.data(), eval_blocks, d_state, lm, PeerLinksOf(links_host_));
            } else if (sharded) {            // fallback: library collective between two kernels
                k_lm_reduce<<<1, 128, 0, stream_>>>(d_partials_.data(), eval_blocks, d_acc_.data());
                AllReduceAccumulator(nccl_comm, d_state);
                k_lm_step<false><<<1, 128, 0, stream_>>>(P, phase, d_acc_.data(), 1, d_state, lm, PeerLinks{});
                launches_ += 1;
            } else {
                k_lm_step<false><<<1, 128, 0, stream_>>>(P, phase, d_partials_.data(), eval_blocks, d_state, lm, PeerLinks{});
            }
            launches_ += 2;
        };
        if (sharded) {   // all-gather of the per-rank valid counts (as a sum of one-hot vectors)
            k_lm_select<<<1, 1024, 0, stream_>>>(P, 1, d_num_keypoints, blocks_buf, d_lm_sel_.data(), d_state, lm, stats, d_acc_.data());
            AllReduceAccumulator(nccl_comm, d_state);
            launches_ += 1;
        }
        k_lm_select<<<1, 1024, 0, stream_>>>(P, 0, d_num_keypoints, blocks_buf, d_lm_sel_.data(), d_state, lm, stats, d_acc_.data());
        launches_ += 2;
        eval_and_step(0);
        for (int ls = 0; ls < opt.ls_max_num_iters; ++ls) eval_and_step(1);
        k_lm_finish<<<1, 32, 0, stream_>>>(P, d_state, lm, it);
        launches_ += 1;
    }
    CT_CUDA_CHECK(cudaGetLastError());
    DebugLmTrace(lm);
}

void IcpSolver::EnqueueCeresBatch(const DeviceMap &map, const cticp_icp_options &opt, const cticp_strategy_options &strategy,
                                  int batch, const size_t *h_n, const float4 *d_keypoints, IcpState *d_states) {
    if (!use_persistent_) throw std::logic_error("batched CERES / ROBUST registration needs the persistent loop");
    if (batch < 1) throw std::invalid_argument("batch must be at least 1");
    CheckCeresOptions(map, opt, strategy);
    const bool robust = opt.solver == CTICP_SOLVER_ROBUST;
    const size_t ncn = robust ? 1 : (size_t) opt.num_closest_neighbors;
    size_t total = 0;
    for (int b = 0; b < batch; ++b) total += h_n[b];
    if (total > (size_t) INT32_MAX) throw std::invalid_argument("too many keypoints in one batch");
    // one set of buffers for the batch: problem b's blocks, sel_idx and classes from ncn · (its first keypoint) on
    EnsureLmBuffers(std::max<size_t>(total, 1) * ncn);
    const DistanceStrategy *distance = UploadLmStrategy(map, opt, strategy) ? d_lm_strategy_.data() : nullptr;
    if (robust) CT_CUDA_CHECK(cudaMemsetAsync(d_lm_classes_.data(), 0, total, stream_));   // NEIGHBORHOOD_TYPE::NONE
    std::vector<LmProblem> problems(batch);
    size_t base = 0;
    for (int b = 0; b < batch; ++b) {
        problems[b] = LmProblem{&map, &opt, &strategy, d_keypoints + base, kp_lo_ ? kp_lo_ + base : nullptr, nullptr, h_n[b],
                                d_states + b, d_lm_blocks_.data() + ncn * base, d_lm_sel_.data() + ncn * base,
                                d_lm_classes_.data() + ncn * base, distance};
        base += h_n[b];
    }
    EnqueueCeresGroups(problems.data(), batch);
}

LmProblem IcpSolver::PrepareCeres(const DeviceMap &map, const cticp_icp_options &opt, const cticp_strategy_options &strategy,
                                  const float4 *d_keypoints, const int *d_num_keypoints, size_t k_hint, size_t k_capacity,
                                  IcpState *d_state) {
    CheckCeresOptions(map, opt, strategy);
    const bool robust = opt.solver == CTICP_SOLVER_ROBUST;
    const int ncn = robust ? 1 : opt.num_closest_neighbors;
    EnsureLmBuffers(k_capacity * (size_t) ncn);
    const bool distance_based = UploadLmStrategy(map, opt, strategy);
    if (robust) CT_CUDA_CHECK(cudaMemsetAsync(d_lm_classes_.data(), 0, k_capacity, stream_));   // NEIGHBORHOOD_TYPE::NONE
    return LmProblem{&map, &opt, &strategy, d_keypoints, kp_lo_, d_num_keypoints, k_hint, d_state, d_lm_blocks_.data(),
                     d_lm_sel_.data(), d_lm_classes_.data(), distance_based ? d_lm_strategy_.data() : nullptr};
}

void IcpSolver::EnqueueCeresGroups(const LmProblem *problems, int batch) {
    if (!use_persistent_) throw std::logic_error("batched CERES / ROBUST registration needs the persistent loop");
    if (batch < 1) throw std::invalid_argument("batch must be at least 1");
    // k_lm_persistent's mode (0 = CERES nearest neighbour, 1 = CERES distance-based, 2 = ROBUST): one per launch
    const auto mode_of = [](const LmProblem &p) {
        return p.opt->solver == CTICP_SOLVER_ROBUST ? 2 : (p.strategy->type == CTICP_STRATEGY_DISTANCE_BASED ? 1 : 0);
    };
    const int mode = mode_of(problems[0]);
    for (int b = 1; b < batch; ++b)
        if (mode_of(problems[b]) != mode) throw std::invalid_argument("a grouped LM launch runs problems of one mode");
    // one problem: the solo launch (grid barriers, the table is not read but for its count)
    const bool grouped = batch > 1;
    void *kernel = LmPersistentKernel(mode, false, grouped);
    const size_t smem = grouped ? kLmGroupedShared : sizeof(LmPShared);
    const int coresident = LmCoresident(grouped ? 6 + mode : mode * 2, kernel, smem);
    if (2 * batch > coresident)
        throw CapacityError("batch of " + std::to_string(batch) + " registrations: the device holds " +
                            std::to_string(coresident) + " CTAs of the LM kernel, two per registration needed");
    // table: LmGroup[B] | first_cta[0..B] | the counts of the problems without a device count
    std::vector<size_t> n(batch);
    for (int b = 0; b < batch; ++b) n[b] = problems[b].n;
    std::vector<int> gather(batch);
    BatchGatherCtas(n.data(), batch, coresident, kp_per_cta_, gather.data());
    const size_t cta_off = sizeof(LmGroup) * (size_t) batch, count_off = cta_off + sizeof(int) * (size_t) (batch + 1);
    const size_t bytes = count_off + sizeof(int) * (size_t) batch;
    d_lm_table_.reserve(bytes, stream_);
    h_lm_table_.assign(bytes, 0);
    LmGroup *table = reinterpret_cast<LmGroup *>(h_lm_table_.data());
    int *first_cta = reinterpret_cast<int *>(h_lm_table_.data() + cta_off);
    int *count = reinterpret_cast<int *>(h_lm_table_.data() + count_off);
    const int *d_count = reinterpret_cast<const int *>(d_lm_table_.data() + count_off);
    for (int b = 0; b < batch; ++b) {
        const LmProblem &p = problems[b];
        if (p.n > (size_t) INT32_MAX) throw std::invalid_argument("too many keypoints in one problem");
        LmGroup &e = table[b];
        e.P = MakeLmParams(*p.map, *p.opt, *p.strategy, p.keypoints_lo, 0, 1);
        e.G = LmGatherConfig(*p.map, e.P);
        e.keypoints = p.keypoints;
        count[b] = (int) p.n;
        e.num_keypoints = p.d_num_keypoints ? p.d_num_keypoints : d_count + b;
        e.st = p.d_state;
        e.blocks = p.blocks;
        e.sel_idx = p.sel_idx;
        e.classes = p.classes;
        e.D = p.distance;
        first_cta[b + 1] = first_cta[b] + 1 + gather[b];
    }
    const int grid = first_cta[batch];
    // per group: its LmState (kLmStateStride), its stats line and its barrier words, each area after the B of the one before
    constexpr size_t kGroupBytes = kLmStateStride + sizeof(unsigned long long) * kLmStatsStride + sizeof(unsigned int) * kLmBarrierWords;
    d_lm_groups_.reserve(kGroupBytes * (size_t) batch, stream_);
    char *area = d_lm_groups_.data();
    auto *lm = reinterpret_cast<LmState *>(area);
    auto *stats = reinterpret_cast<unsigned long long *>(area + kLmStateStride * batch);
    auto *barrier = reinterpret_cast<unsigned int *>(area + (kLmStateStride + sizeof(unsigned long long) * kLmStatsStride) * batch);
    EnsurePartials(grid - batch);
    CT_CUDA_CHECK(cudaMemcpyAsync(d_lm_table_.data(), h_lm_table_.data(), bytes, cudaMemcpyHostToDevice, stream_));
    CT_CUDA_CHECK(cudaMemsetAsync(barrier, 0, sizeof(unsigned int) * kLmBarrierWords * batch, stream_));

    // the solo launch takes problem 0's entry as its parameters; the grouped one reads the table only
    GatherConfig G = grouped ? GatherConfig{} : table[0].G;
    LmParams P = grouped ? LmParams{} : table[0].P;
    const float4 *kp = grouped ? nullptr : table[0].keypoints;
    const int *nk = grouped ? nullptr : table[0].num_keypoints;
    IcpState *st = grouped ? nullptr : table[0].st;
    ResidualBlock *blocks_buf = grouped ? nullptr : table[0].blocks;
    int *sel = grouped ? nullptr : table[0].sel_idx;
    unsigned char *classes = grouped ? nullptr : table[0].classes;
    const DistanceStrategy *dstrat = grouped ? nullptr : table[0].D;
    double *parts = d_partials_.data();
    PeerLinks links{};
    LmGroups groups = grouped ? LmGroups{reinterpret_cast<const LmGroup *>(d_lm_table_.data()), batch, barrier} : LmGroups{};
    void *args[] = {&G, &P, &kp, &nk, &st, &lm, &blocks_buf, &sel, &classes, &stats, &dstrat, &parts, &links, &groups};
    const bool timed = time_gather_ && ev_used_ < kMaxEvents;
    if (timed) cudaEventRecord(ev_begin_[ev_used_].get(), stream_);
    CT_CUDA_CHECK(cudaLaunchCooperativeKernel(kernel, dim3(grid), dim3(kLmPWarps * 32), args, smem, stream_));
    if (timed) cudaEventRecord(ev_end_[ev_used_++].get(), stream_);
    gather_launches_ += 1;
    launches_ += 1;
}

void IcpSolver::DebugLmTrace(void *d_lm) {
    const bool timers = getenv("CTICP_DEBUG_TIMERS") != nullptr;
    if (!getenv("CTICP_DEBUG_LM") && !timers) return;
    static LmState h;
    CT_CUDA_CHECK(cudaMemcpyAsync(&h, d_lm, sizeof(LmState), cudaMemcpyDeviceToHost, stream_));
    CT_CUDA_CHECK(cudaStreamSynchronize(stream_));
    if (timers) {
        const unsigned long long *c = h.dbg_cycles;
        fprintf(stderr, "[cticp] LM loop, solver CTA (SM cycles, needs a -DCTICP_DEBUG_TIMERS build): loop %llu = assembly wait %llu + "
                "selection %llu + evaluation wait %llu + reduce %llu + minimizer step %llu + barriers %llu; %llu evaluations\n",
                c[0], c[1], c[2], c[3], c[4], c[5], c[6], c[7]);
        if (!getenv("CTICP_DEBUG_LM")) return;
    }
    for (int i = 0; i < h.trace_n; ++i)
        fprintf(stderr, "[eng-lm] x_cost %.12g cand %.12g x %.12g %.12g %.12g %.12g | %.12g %.12g %.12g %s\n", h.trace[i][0], h.trace[i][1],
                h.trace[i][6], h.trace[i][7], h.trace[i][8], h.trace[i][9], h.trace[i][10], h.trace[i][11], h.trace[i][12], h.trace[i][5] > 0.5 ? "ACCEPT" : "reject");
}

}  // namespace cticp
