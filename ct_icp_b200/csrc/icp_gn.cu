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
#include "gn_step.cuh"
#include "peer_exchange.cuh"
#include "small_solve.cuh"
#include "tagged_words.cuh"

namespace cticp {
namespace cg = cooperative_groups;

// Warps per CTA of the gather kernels (one keypoint per warp at a time). Fewer, fatter CTAs make the grid-wide
// barriers and the reduction of the per-CTA partial sums cheaper, and more warps share one SM's instruction cache: on
// config 2 (K ~ 1.2k) the GN loop per frame got faster from 4 to 8 to 16 warps (CTICP_GATHER_WARPS selects it)
// (16 warps x 128 registers = the whole register file: one CTA per SM, ~77 CTAs).
#ifndef CTICP_GATHER_WARPS
#define CTICP_GATHER_WARPS 16
#endif
constexpr int kGatherWarps = CTICP_GATHER_WARPS;

// The warp-specialised layout of the single-GPU k_gn_persistent (gn_ws_loop): six warpgroups, 768 threads. Warpgroups
// 0-4 are gather warps (phase B only), warpgroup 5 the math warps (the pose, phases A and C one keypoint per lane, and
// in the solver CTA the 12x12 solve). setmaxnreg moves registers from the gather warps to the math warps: 80 per thread
// at launch (65536 / 768, in steps of 8), then 72 for the gather warps and 120 for the math warps — 20 x 32 x 72 +
// 4 x 32 x 120 = 768 x 80, the CTA's allocation at launch.
constexpr int kWsGatherWarps = 20;
constexpr int kWsMathWarps = 4;
constexpr int kWsWarps = kWsGatherWarps + kWsMathWarps;
#ifndef CTICP_WS_GATHER_REGS
#define CTICP_WS_GATHER_REGS 72
#endif
constexpr int kWsGatherRegs = CTICP_WS_GATHER_REGS;
constexpr int kWsMathRegs = (kWsWarps * 80 - kWsGatherWarps * kWsGatherRegs) / kWsMathWarps;
static_assert(kWsGatherWarps % 4 == 0 && kWsMathWarps == 4 && kWsGatherWarps >= kGatherWarps, "warpgroups");
static_assert(kWsMathRegs <= 256 && kWsMathRegs % 8 == 0, "setmaxnreg");
// phase A of one keypoint: its world position and voxel
struct WsQuery {
    double x, y, z;
    int kx, ky, kz;
};



struct GatherLaunch {
    GatherConfig G;
    GnParams P;
};

// One registration of a grouped k_gn_persistent launch (GnGroups): everything a solo launch takes as kernel parameters.
// Groups may search different maps with different options (the odometry's batch: one handle per group).
struct GnGroup {
    GatherLaunch cfg;            // map level, search and GN parameters; cfg.P.kp_lo: the group's residual plane
    const float4 *keypoints;
    const int *num_keypoints;    // device count
    IcpState *st;
    int num_iters;
};

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
// warps had no tile at all. The exception (gn_pair_schedule): in the sharded k_gn_persistent, a range of more keypoints than warps but
// at most two per warp gets one tile per warp from the last iteration's costs (the first iteration: in keypoint order) —
// the heaviest keypoints alone, the others in pairs — instead of a few warps running a second whole chain after their
// first.
struct GnPose {
    Q4 qb, qe;
    V3 tb, te;
    SlerpConsts sc;
};
struct GnWarpAcc {
    double sum_sq = 0;               // (unused: Σ scalar² comes out of the CTA's row reduction, accumulator kAccSumSq)
    unsigned n_stencil = 0;          // per-lane partial counters
    int n_used = 0, n_kp = 0, n_valid = 0;
    CT_STAMP(long long dbg[5] = {0, 0, 0, 0, 0};)   // cycles in phases A, B, C; end of the warp's last tile; longest tile
};
constexpr int kDbgIters = 8, kDbgSlots = 8;

constexpr int kTileMax = 16;   // keypoints per warp tile (phases A / C cost 1/W per keypoint: 16 is deep in the flat part)
constexpr int kRowCap = 256;   // rows of a CTA's range held in shared memory at a time (longer ranges go in chunks)
constexpr int kRowParts = 5;   // the row reduction splits the rows over 5 x 96 threads

// The moments of one keypoint as phase B hands them to phase C: [0] the kept neighbours (low word) and the stencil points
// (high word) — two integers in one slot, no int <-> double conversion —, [1..12] s*, f* of NeighborSums (only when at
// least `need` neighbours were kept). As wide as a row of CtaRows::u, which the warp-specialised loop stores them in.
constexpr int kMomentWords = 13;
__device__ __forceinline__ void gn_store_moments(double *o, const NeighborSums &s, unsigned spts, int need) {
    o[0] = __hiloint2double((int) spts, s.n);
    if (s.n >= need) {
        o[1] = s.sx; o[2] = s.sy; o[3] = s.sz;
        o[4] = s.sxx; o[5] = s.sxy; o[6] = s.sxz; o[7] = s.syy; o[8] = s.syz; o[9] = s.szz;
        o[10] = s.fx; o[11] = s.fy; o[12] = s.fz;
    }
}
__device__ __forceinline__ unsigned moments_stencil_points(const double *o) { return (unsigned) __double2hiint(o[0]); }

// ---- A: world_kpts[i] = InterpolatePose(begin, end, t_i) * raw_i  (ct_icp.cpp:964-966, types.h:361-366): the world
// position of a keypoint (`kraw`: raw xyz in the sensor frame + alpha timestamp, load_raw) and its voxel. Every schedule
// calls this one function, so the arithmetic is one instruction sequence.
__device__ __forceinline__ void gn_phase_a(const GatherConfig &G, const RawPoint &kraw, const GnPose &pose, bool rigid,
                                           double inv_res, V3 &p, int &kx, int &ky, int &kz) {
    const V3 raw{kraw.x, kraw.y, kraw.z};
    p = rigid ? qrot(qnormalized(pose.qe), raw) + pose.te
              : ct_transform_c(pose.qb, pose.tb, pose.qe, pose.te, kraw.alpha, raw, pose.sc);
    kx = query_voxel_coord(p.x, G.L.res, inv_res);
    ky = query_voxel_coord(p.y, G.L.res, inv_res);
    kz = query_voxel_coord(p.z, G.L.res, inv_res);
    confine_query(kx, ky, kz, G.r);
}

// ---- C (ct_icp.cpp:769-850): a keypoint's moments `o` (world position p) → covariance, closed-form eigen, normal, a2D,
// residual and 12-vector Jacobian row u[0..12]; returns whether the row is used. `raw()` gives the keypoint's RawPoint
// (called only for a used row). `o` may alias `u`: every moment is read before the first store. Every schedule calls
// this one function.
template <class RawFn>
__device__ __forceinline__ bool gn_phase_c(const GnParams &P, RawFn raw, const GnPose &pose, const V3 &p, int need,
                                           const double *o, double *u, GnWarpAcc &A) {
    bool used = false;
    NeighborSums mine;
    mine.n = __double2loint(o[0]);
    A.n_kp += 1;
    A.n_stencil += moments_stencil_points(o);
    if (mine.n >= need) {
        A.n_valid += 1;
        mine.sx = o[1]; mine.sy = o[2]; mine.sz = o[3];
        mine.sxx = o[4]; mine.sxy = o[5]; mine.sxz = o[6]; mine.syy = o[7]; mine.syz = o[8]; mine.szz = o[9];
        mine.fx = o[10]; mine.fy = o[11]; mine.fz = o[12]; mine.fd2 = 0;
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
            const RawPoint kraw = raw();
            const V3 xyz{kraw.x, kraw.y, kraw.z};
            const V3 ob = qrot(pose.qb, xyz), oe = qrot(pose.qe, xyz);   // :813-816
            const double a = kraw.alpha, am = 1.0 - a;
            const V3 cb = cross(ob, nw), ce = cross(oe, nw);
            u[0] = am * cb.x; u[1] = am * cb.y; u[2] = am * cb.z;
            u[3] = am * nw.x; u[4] = am * nw.y; u[5] = am * nw.z;
            u[6] = a * ce.x;  u[7] = a * ce.y;  u[8] = a * ce.z;
            u[9] = a * nw.x;  u[10] = a * nw.y; u[11] = a * nw.z;
            u[12] = -scalar;   // b -= u * scalar (:849)
            used = true;
            A.n_used += 1;
        }
    }
    return used;
}

// Per-warp shared memory of a tile: the gather's staging area and the moments of each keypoint of the tile (phase B hands
// them to phase C through here instead of through 27 registers that would stay live across the gather).
struct __align__(16) TileScratch {
    SelScratch sel;
    double sums[kTileMax][kMomentWords];
};
// Per-CTA row table of the current chunk of the CTA's range
struct __align__(16) CtaRows {
    double u[kRowCap][13];       // u[0..11], -scalar of keypoint (chunk base + r); valid iff used[r]
    unsigned char used[kRowCap];
    double red[kRowParts][kAcc];
    int next;                    // tile counter of the chunk
    // the paired schedule (gn_pair_schedule): stencil points of keypoint r in the last iteration (written for every range:
    // no bound check in phase C), and this iteration's tiles — warp w takes pair[w][0] and pair[w][1] (kNoKeypoint: none)
    unsigned cost[kRowCap];
    unsigned char pair[kGatherWarps][2];
};
constexpr unsigned char kNoKeypoint = 0xff;

// keypoints per tile for a CTA range of `span` keypoints
__device__ __forceinline__ int gn_tile_width(int span) {
    // one keypoint per grab while the range is at most two rounds of the CTA's warps (the loop is bound by the slowest
    // keypoint there: balance counts); beyond that one tile per warp, as wide as it gets (throughput: the lane-per-keypoint
    // phases cost 1/W per keypoint — on the dense workload, K = 32k, tiles of 7 were slower than tiles of 14)
    if (span <= 2 * CTICP_GATHER_WARPS) return 1;
    const int W = (span + CTICP_GATHER_WARPS - 1) / CTICP_GATHER_WARPS;
    return W < kTileMax ? W : kTileMax;
}

// ranges that take the paired schedule once the last iteration's costs are known: more keypoints than warps, at most two
// per warp (one keypoint per lane of the warp that builds the schedule: CTAs of at most 16 warps)
__device__ __forceinline__ bool gn_pairs_apply(int span) {
    return kGatherWarps > 1 && 2 * kGatherWarps <= 32 && span > kGatherWarps && span <= 2 * kGatherWarps;
}

// The static schedule of a range of kGatherWarps < n <= 2 kGatherWarps keypoints from the costs of the last iteration
// (R.cost[0..n), written by every keypoint's phase C): one tile per warp, S = 2 kGatherWarps - n single tiles and
// n - kGatherWarps pairs. The S heaviest keypoints (most stencil points; ties: lower index first) get a warp each and the
// remaining ones are paired heaviest with lightest, which makes the largest pair cost as small as it can be (the first
// iteration has no costs: all zero, the order is the keypoint order). A pair runs
// phases A and C once for both keypoints (lanes 0 and 1) instead of a second whole chain on the warp that grabbed it.
// The schedule is a function of the costs alone; the rows go to R.u by keypoint as before, so the result does not depend
// on it. One warp; writes R.pair.
__device__ __noinline__ void gn_pair_schedule(CtaRows &R, int n, int lane) {
    const unsigned c = lane < n ? R.cost[lane] : 0u;
    int rank = 0;   // position in the order heaviest first, lower index first among equals
    for (int j = 0; j < n; ++j) {
        const unsigned cj = __shfl_sync(0xffffffffu, c, j);
        rank += (cj > c || (cj == c && j < lane)) ? 1 : 0;
    }
    const int singles = 2 * kGatherWarps - n, pairs = n - kGatherWarps;
    if (lane < n) {
        if (rank < singles) {
            R.pair[rank][0] = (unsigned char) lane;
            R.pair[rank][1] = kNoKeypoint;
        } else if (rank < singles + pairs) {
            R.pair[rank][0] = (unsigned char) lane;
        } else {
            R.pair[singles + (n - 1 - rank)][1] = (unsigned char) lane;
        }
    }
}

// The tiles of the chunk [lo, hi) of this CTA's range (hi - lo <= kRowCap); R.next must be 0 and visible (barrier) on entry.
// `pair` (nullptr: tiles of W keypoints grabbed from R.next): this warp's one tile of the paired schedule (R.pair).
__device__ __forceinline__ void gn_gather_tiles(const GatherConfig &G, const GnParams &P, const int *stencil,
                                                const float4 *__restrict__ keypoints, int lo, int hi, int W,
                                                const unsigned char *pair, const GnPose &pose, TileScratch &T,
                                                CtaRows &R, int lane, GnWarpAcc &A, void *bulk = nullptr,
                                                bool rigid = false) {
    if (hi <= lo) return;
    const int need = P.kmin > 5 ? P.kmin : 5;   // ct_icp.cpp:769 ; neighborhood.h:227
    const double inv_res = 1.0 / G.L.res;

    for (bool first = true;; first = false) {
        int wt, r;   // keypoints of the tile; lane < wt: the row (keypoint lo + r) of lane's keypoint
        if (pair) {
            if (!first) break;
            wt = pair[1] == kNoKeypoint ? 1 : 2;
            r = pair[lane == 0 ? 0 : 1];
        } else {
            int j0 = 0;
            if (lane == 0) j0 = atomicAdd(&R.next, W);
            j0 = __shfl_sync(0xffffffffu, j0, 0);
            if (lo + j0 >= hi) break;
            wt = (hi - lo - j0) < W ? (hi - lo - j0) : W;
            r = j0 + lane;
        }
        CT_STAMP(const long long t_a = clock64();)
        V3 p{0, 0, 0};
        int kx = 0, ky = 0, kz = 0;
        if (lane < wt) gn_phase_a(G, load_raw(keypoints, P.kp_lo, lo + r), pose, rigid, inv_res, p, kx, ky, kz);
        CT_STAMP(const long long t_b = clock64();)
        // ---- B
        for (int j = 0; j < wt; ++j) {
            const V3 q{__shfl_sync(0xffffffffu, p.x, j), __shfl_sync(0xffffffffu, p.y, j), __shfl_sync(0xffffffffu, p.z, j)};
            const int qx = __shfl_sync(0xffffffffu, kx, j), qy = __shfl_sync(0xffffffffu, ky, j),
                      qz = __shfl_sync(0xffffffffu, kz, j);
            NeighborSums s;
            unsigned spts = 0;
            warp_gather_sums<false>(G, P.bucket_scale, stencil, q, qx, qy, qz, need, lane, T.sel, s, spts, V3{0, 0, 0}, bulk);
            if (lane == 0) gn_store_moments(T.sums[j], s, spts, need);
        }
        __syncwarp();
        CT_STAMP(const long long t_c = clock64();)
        if (lane < wt) {
            const unsigned spts = moments_stencil_points(T.sums[lane]);
            R.cost[r] = spts;   // the next iteration's schedule (gn_pair_schedule)
            const auto raw = [&] { return load_raw(keypoints, P.kp_lo, lo + r); };
            R.used[r] = gn_phase_c(P, raw, pose, p, need, T.sums[lane], R.u[r], A) ? 1 : 0;
        }
        __syncwarp();   // the moments are consumed before the next tile rewrites them
        CT_STAMP(const long long t_e = clock64();
                 A.dbg[0] += t_b - t_a; A.dbg[1] += t_c - t_b; A.dbg[2] += t_e - t_c;
                 A.dbg[3] = t_e; if (t_e - t_a > A.dbg[4]) A.dbg[4] = t_e - t_a;)
    }
}

// A += u u^T, b -= u scalar over the rows [0, n) of the chunk, in keypoint order within each of kRowParts interleaved
// classes, the classes then in fixed order: deterministic whatever warp wrote a row. Thread t < kRowParts * kAcc handles
// accumulator t % kAcc (entries 0..89: pairs of [A upper | b]; 90: rows used; 91: Σ scalar²) of class t / kAcc. The sum
// of the chunk is ADDED to `carry` of the threads < kAcc. Called by all threads of the CTA; barriers inside.
// `sync` is the CTA-wide barrier (the warp-specialised loop: gn_ws_sync, called by its math warps as well).
struct GnCtaSync {
    __device__ __forceinline__ void operator()() const { __syncthreads(); }
};
template <class Sync = GnCtaSync>
__device__ __forceinline__ void gn_cta_reduce_rows(CtaRows &R, int n, double &carry, Sync sync = Sync{}) {
    const int t = threadIdx.x;
    const int a = t % kAcc, part = t / kAcc;
    sync();   // every row of the chunk is written
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
    sync();
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
    union {
        TileScratch tile[kGatherWarps];   // one warp per tile of keypoints (k_gn_iterate, the sharded k_gn_persistent)
        struct {                          // the warp-specialised k_gn_persistent (gn_ws_loop)
            SelScratch sel[kWsGatherWarps];   // staging area of each gather warp
            WsQuery q[kRowCap];               // phase A of row r of the chunk, for phases B and C
        } ws;
    };
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
    struct {          // k_gn_persistent: the group's words, read where used (no registers held across the gather)
        IcpState *st;
        unsigned long long *rows;   // tagged partial rows: gather CTA, its own; solver CTA, the group's first
        unsigned long long *pose;   // the group's tagged pose words
        int gather_ctas;
    } grp;
    GnGroup group;    // k_gn_persistent: this CTA's entry of the group table (solo: the kernel parameters)
    unsigned long long mbar[kGatherWarps];   // -DCTICP_SEL_BULK: one mbarrier per warp for the bulk copies
};

// the per-warp column sums of a row reduction (columns lane, lane + 32, lane + 64) → their sum in warp order in
// sh.acc[0][0..kAcc). Called by all threads, after a barrier that follows every earlier read of sh.acc.
// Warps w >= kGatherWarps (the warp-specialised solver CTA) have no partials and only join the barriers.
template <class Sync = GnCtaSync>
__device__ __forceinline__ void gn_sum_warp_partials(GnShared &sh, double a0, double a1, double a2, int lane, int w,
                                                     Sync sync = Sync{}) {
    if (w < kGatherWarps) {
        sh.acc[w][lane] = a0;
        sh.acc[w][lane + 32] = a1;
        sh.acc[w][lane + 64] = a2;
    }
    sync();
    double sum = 0;
    if (threadIdx.x < kAcc) {
#pragma unroll
        for (int ww = 0; ww < kGatherWarps; ++ww) sum += sh.acc[ww][threadIdx.x];
    }
    sync();
    if (threadIdx.x < kAcc) sh.acc[0][threadIdx.x] = sum;
    sync();
}

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
    gn_sum_warp_partials(sh, a0, a1, a2, lane, w);
}

// The gather half of an iteration for one CTA: its range [c_lo, c_hi) of the keypoints, in chunks of kRowCap rows →
// the CTA's partial row (kAcc doubles): thread t < kAcc returns entry t. On entry sh.pose is valid and sh.rows.next == 0,
// both visible to the CTA (the thread that fetched the pose set them before a barrier). `paired`: sh.rows.pair holds the
// schedule of this range (gn_pair_schedule; only for gn_pairs_apply ranges, which are one chunk). All threads call.
__device__ __forceinline__ double gn_cta_gather(const GatherConfig &G, const GnParams &P, const int *stencil,
                                                const float4 *__restrict__ keypoints, int c_lo, int c_hi, GnShared &sh,
                                                int lane, int w, GnWarpAcc &A, void *bulk, bool rigid, bool paired = false) {
    const int W = gn_tile_width(c_hi - c_lo);
    const unsigned char *pair = paired ? sh.rows.pair[w] : nullptr;
    double carry = 0;
    for (int base = c_lo;; base += kRowCap) {
        const int top = (c_hi - base) > kRowCap ? base + kRowCap : c_hi;
        gn_gather_tiles(G, P, stencil, keypoints, base, top, W, pair, sh.pose, sh.tile[w], sh.rows, lane, A, bulk, rigid);
        gn_cta_reduce_rows(sh.rows, top > base ? top - base : 0, carry);
        if (top >= c_hi) break;
        if (threadIdx.x == 0) sh.rows.next = 0;
        __syncthreads();
    }
    gn_store_warp_row(sh.acc[w], A, lane);
    __syncthreads();
    const int t = threadIdx.x;
    double s = 0;
    if (t <= kAccSumSq) s = carry;
    else if (t == kAccStencil || t == kAccKeypoints || t == kAccValidNb) {
#pragma unroll
        for (int ww = 0; ww < kGatherWarps; ++ww) s += sh.acc[ww][t];
    }
    return s;
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
        const double s = gn_cta_gather(cfg.G, cfg.P, stencil, keypoints, c_lo, c_hi, sh, lane, w, A, bulk_ptr,
                                       active && P.rigid_first && __ldcg(&st->iter) == 0);
        if (threadIdx.x < kAcc) __stcg(partials + (size_t) blockIdx.x * kAcc + threadIdx.x, s);
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

// ---- synchronisation of the persistent loop: tagged words (tagged_words.cuh), no fence, no flag, no atomic ---------------
// The loop's dependencies are asymmetric: the solver CTA needs every gather CTA's partial row; a gather CTA needs the solver
// CTA's new pose and `done` flag — it never needs the OTHER gather CTAs. Both hand-offs are tagged words:
//  - a gather CTA stores its row of iteration `it` as 2 x kAcc words tagged `tag + it` (each double as its two 32-bit
//    halves) and goes straight on to wait for the next pose; the solver CTA's warps consume the rows in a fixed order, each
//    as soon as its words carry that tag (gn_reduce_tagged_rows), so the reduction ends about one L2 trip after the last
//    row lands;
//  - after the solve the solver warp publishes the pose pair, the slerp constants and `done` as kPosePairs word pairs
//    tagged `tag + it + 1`; warp 0 of a gather CTA polls them until every pair carries that tag: the poll is the fetch.
// One buffer per direction is enough. A gather CTA rewrites its row only after it has read the next pose, which the solver
// publishes only after it has consumed every row of the iteration; the solver rewrites the pose words only after every row
// of the next iteration has arrived, i.e. after every gather CTA has read them. Tags come from a per-solver counter
// (IcpSolver::ReserveLoopTags): a launch reserves num_iters + 1 consecutive values and the words are zeroed when allocated
// and before the counter wraps, so a word left by another iteration or launch never carries the tag a poll waits for.
// Iteration 0 reads the state the host uploaded; the full IcpState goes to `st` once, when the solver CTA leaves the loop.
// The launch stays cooperative: the CTAs must be co-resident for the polls to make progress. Every poll is bounded: a
// protocol error ends the kernel with st->failed = 2 instead of hanging the device.
#ifndef CTICP_GN_GRID_BARRIERS
#define CTICP_GN_FLAG_SYNC 1
#endif
// threads of a k_gn_persistent CTA: the warp-specialised layout (gn_ws_loop) for the single-GPU loop, one warp per tile of
// keypoints for the sharded one (and for the -DCTICP_GN_GRID_BARRIERS variant)
constexpr int gn_persistent_threads(bool peers) {
#ifdef CTICP_GN_FLAG_SYNC
    return peers ? kGatherWarps * 32 : kWsWarps * 32;
#else
    return (void) peers, kGatherWarps * 32;
#endif
}
constexpr int kRowWords = 2 * kAcc;   // tagged words of a partial row
// pose words of a group: the bytes of GnPose as 32-bit halves, then `done` (and an unused half), in word pairs
constexpr int kPosePairs = 18;
constexpr int kPoseGroupWords = 48;   // one group's pose words (three 128-byte lines)
static_assert(sizeof(GnPose) == 8 * (kPosePairs - 1) && 2 * kPosePairs <= kPoseGroupWords, "pose words");
struct GnLoopWords {
    unsigned long long *rows;   // partial rows of the gather CTAs, kRowWords each (group g's after those of groups < g)
    unsigned long long *pose;   // kPoseGroupWords per group
    unsigned int tag;           // tag of iteration 0's rows; iteration it's rows and pose words carry tag + it
};

// The groups of one grouped k_gn_persistent launch (k_gn_persistent<false, true>). Group g owns the CTAs
// [first_cta[g], first_cta[g + 1]) of the grid — the first is g's solver CTA, the others gather g's keypoints — the
// registration table[g], the partial rows [first_cta[g] - g, first_cta[g + 1] - g - 1) and its own pose words. Groups
// never wait on each other. Both arrays are in device memory (IcpSolver::EnqueueGaussNewtonGroups).
struct GnGroups {
    const GnGroup *table;        // [num_groups]
    const int *first_cta;        // [num_groups + 1]
    int num_groups;
};

// The solver CTA's reduction of the `n` tagged rows of iteration `tag`, bit for bit the sum of gn_reduce_rows: warp w
// consumes its rows w, w + kGatherWarps, … in that order, each as soon as its words carry the tag (the rows land over the
// whole gather, so most are added before the last one arrives); then the per-warp sums in warp order. Result in
// sh.acc[0][0..kAcc). Returns false (uniform) when a row has not arrived within kLoopSyncTimeout. Called by all threads.
// One row per warp at a time: loads of more rows in flight need registers that this kernel's gather path then spills to
// local memory (on the bench workload the GN launch took 161 us with five rows in flight, 157 us with two, 151 us with one).
// warp w < kGatherWarps: its rows of the reduction below, summed into a0..a2; false when one did not arrive in time
__device__ __forceinline__ bool gn_consume_tagged_rows(const unsigned long long *rows, int n, unsigned int tag, int lane,
                                                       int w, double &a0, double &a1, double &a2) {
    bool ok = true;
    const long long t0 = clock64();
    for (int b = w; b < n && ok; b += kGatherWarps) {
        const unsigned long long *row = rows + (size_t) b * kRowWords + 2 * lane;
        ulonglong2 c0, c1, c2;
        while (true) {
            c0 = tagged_load_u64x2(row);
            c1 = tagged_load_u64x2(row + 64);
            c2 = tagged_load_u64x2(row + 128);
            if (pair_tagged(c0, tag) && pair_tagged(c1, tag) && pair_tagged(c2, tag)) break;
            if (clock64() - t0 > kLoopSyncTimeout) {
                ok = false;
                break;
            }
        }
        if (ok) {
            a0 += pair_double(c0);
            a1 += pair_double(c1);
            a2 += pair_double(c2);
        }
    }
    return ok;
}
__device__ __forceinline__ bool gn_reduce_tagged_rows(GnShared &sh, const unsigned long long *rows, int n, unsigned int tag,
                                                      int lane, int w) {
    double a0 = 0, a1 = 0, a2 = 0;
    const bool ok = gn_consume_tagged_rows(rows, n, tag, lane, w, a0, a1, a2);
    if (!__syncthreads_and(ok)) return false;
    gn_sum_warp_partials(sh, a0, a1, a2, lane, w);
    return true;
}

// solver warp: the pose words of the next iteration, tagged `tag`, from the working state (GnPose's layout, then `done`)
__device__ __forceinline__ void gn_publish_pose(unsigned long long *words, const IcpState &s, unsigned int tag, int lane) {
    if (lane >= kPosePairs) return;
    unsigned int lo, hi;
    if (lane < 16) {
        const double *d = lane < 4 ? s.qb + lane : lane < 8 ? s.qe + (lane - 4) : lane < 11 ? s.tb + (lane - 8)
                        : lane < 14 ? s.te + (lane - 11) : lane == 14 ? &s.slerp_theta : &s.slerp_inv_sin;
        lo = (unsigned int) __double2loint(*d);
        hi = (unsigned int) __double2hiint(*d);
    } else if (lane == 16) {
        lo = (unsigned int) s.slerp_linear;
        hi = (unsigned int) s.slerp_negate;
    } else {
        lo = (unsigned int) s.done;
        hi = 0;
    }
    tagged_store_u64x2(words + 2 * lane, tagged_word(tag, lo), tagged_word(tag, hi));
}

// warp 0 of a gather CTA: polls the pose words until every pair carries `tag`, then → sh.pose / sh.done (a poll that runs
// out of time reads as done: the CTA leaves the loop)
__device__ __forceinline__ void gn_fetch_pose(GnShared &sh, unsigned int tag, long long timeout, int lane) {
    const unsigned long long *src = sh.grp.pose + 2 * lane;
    const bool mine = lane < kPosePairs;
    ulonglong2 v = make_ulonglong2(0ull, 0ull);
    const long long t0 = clock64();
    bool ok = true;
    while (true) {
        if (mine) v = tagged_load_u64x2(src);
        if (__all_sync(0xffffffffu, !mine || pair_tagged(v, tag))) break;
        if (__any_sync(0xffffffffu, clock64() - t0 > timeout)) {
            ok = false;
            break;
        }
    }
    if (lane < kPosePairs - 1) {
        unsigned int *dst = reinterpret_cast<unsigned int *>(&sh.pose) + 2 * lane;
        dst[0] = word_payload(v.x);
        dst[1] = word_payload(v.y);
    } else if (lane == kPosePairs - 1)
        sh.done = ok ? (int) word_payload(v.x) : 1;
}

// ---- the warp-specialised loop of the single-GPU k_gn_persistent (kWsWarps warps: kWsGatherWarps gather warps, then the
// kWsMathWarps math warps) -------------------------------------------------------------------------------------------------
// From the setmaxnreg on, the two roles run separate code to the end of the kernel (ptxas gives a region the registers of
// the setmaxnreg that leads to it only where the roles do not merge again) and meet at named barrier 1 of all kWsWarps
// warps, which either role reaches from its own code: every barrier of one role has its partner in the other.
// Per chunk of a gather CTA's range (kRowCap rows):
//   math warps, thread m : phase A of rows m, m + 128 → sh.ws.q (first chunk: after the pose) | barrier
//   gather warps         : phase B, one row per grab from sh.rows.next (no pairs while the range is at most
//                          kWsGatherWarps rows: the bench's ranges are 18-20) → the row's moments in sh.rows.u | barrier
//   math warps           : phase C of the same rows, the moments in sh.rows.u replaced by the row
//   gather warps         : gn_cta_reduce_rows (barriers inside; the math warps join them)
// The rows are the rows of gn_gather_tiles (one gn_phase_a / gn_phase_c) and their reduction is the same, so the partial
// row is the same bit for bit. The solver CTA: gather warps 0..kGatherWarps-1 consume the tagged rows as
// gn_reduce_tagged_rows does, the first math warp solves and publishes the pose (the registers are there).
struct GnWsSync {
    __device__ __forceinline__ void operator()() const {
        asm volatile("barrier.sync 1, %0;" ::"n"(kWsWarps * 32) : "memory");
    }
};
__device__ __forceinline__ bool gn_ws_sync_and(bool pred) {
    unsigned r;
    asm volatile("{\n.reg .pred p, q;\nsetp.ne.u32 p, %1, 0;\nbarrier.red.and.pred q, 1, %2, p;\nselp.u32 %0, 1, 0, q;\n}"
                 : "=r"(r) : "r"((unsigned) pred), "n"(kWsWarps * 32) : "memory");
    return r != 0;
}

// gather CTA, gather warp w: phase B of every chunk of every iteration, the reduction of the rows, the tagged partial row
__device__ __forceinline__ void gn_ws_gather_warp(GnShared &sh, const GatherConfig &G, const int *stencil, int num_iters,
                                                  int c_lo, int c_hi, unsigned int tag0, int lane, int w) {
    const GnWsSync sync;
    const GnParams &P = sh.group.cfg.P;
    const int need = P.kmin > 5 ? P.kmin : 5;   // ct_icp.cpp:769 ; neighborhood.h:227
    CtaRows &R = sh.rows;
    for (int it = 0; it < num_iters; ++it) {
        // (CTICP_DEBUG_FLAGS & 2, timing only: an empty range — the hand-off and the reduction without the gather work)
        const bool skip = (P.debug_flags & 2) != 0;
        const int lo = skip ? 0 : c_lo, hi = skip ? 0 : c_hi;
        double carry = 0;
        bool done = false;
        for (int base = lo;; base += kRowCap) {
            const int top = (hi - base) > kRowCap ? base + kRowCap : hi;
            const int n = top > base ? top - base : 0;
            sync();   // phase A of the chunk (the first chunk: also the pose and `done`)
            if (sh.done) {
                done = true;
                break;
            }
            while (true) {
                int r = 0;
                if (lane == 0) r = atomicAdd(&R.next, 1);
                r = __shfl_sync(0xffffffffu, r, 0);
                if (r >= n) break;
                const WsQuery &q = sh.ws.q[r];
                NeighborSums s;
                unsigned spts = 0;
                warp_gather_sums<false>(G, P.bucket_scale, stencil, V3{q.x, q.y, q.z}, q.kx, q.ky, q.kz, need, lane,
                                        sh.ws.sel[w], s, spts);
                if (lane == 0) gn_store_moments(R.u[r], s, spts, need);
            }
            sync();   // phase B of the chunk
            gn_cta_reduce_rows(R, n, carry, sync);   // (the math warps' counters are in sh.acc from its first barrier on)
            if (top >= hi) break;
            if (threadIdx.x == 0) R.next = 0;
            sync();
        }
        if (done) break;
        const int t = threadIdx.x;
        if (t < kAcc) {
            double s = 0;
            if (t <= kAccSumSq) s = carry;
            else if (t == kAccStencil || t == kAccKeypoints || t == kAccValidNb) {
#pragma unroll
                for (int ww = 0; ww < kWsMathWarps; ++ww) s += sh.acc[ww][t];
            }
            tagged_store_double(sh.grp.rows + 2 * t, tag0 + (unsigned int) it, s);
        }
        if (it == num_iters - 1) break;   // nothing left to wait for: the solver CTA finishes the registration alone
    }
}

// math warps only (named barrier 2): the pose and `done` that the first math warp fetched
__device__ __forceinline__ void gn_ws_math_sync() {
    asm volatile("barrier.sync 2, %0;" ::"n"(kWsMathWarps * 32) : "memory");
}
constexpr int kWsRowsPerLane = kRowCap / (kWsMathWarps * 32);   // rows of a chunk per math thread
static_assert(kWsRowsPerLane * kWsMathWarps * 32 == kRowCap, "rows per math thread");

// gather CTA, math warp mw = w - kWsGatherWarps: the pose, phases A and C, the per-keypoint counters. Thread m does rows
// m + 128 j of a chunk; their raw keypoints are loaded into registers before the pose is waited for (the range is the
// same in every iteration), so neither phase waits for a keypoint load in the first chunk.
__device__ __forceinline__ void gn_ws_gather_math(GnShared &sh, const GatherConfig &G, int num_iters, int c_lo, int c_hi,
                                                  unsigned int tag0, int lane, int w) {
    const GnWsSync sync;
    const GnParams &P = sh.group.cfg.P;
    const float4 *__restrict__ keypoints = sh.group.keypoints;
    const int need = P.kmin > 5 ? P.kmin : 5;
    const int mw = w - kWsGatherWarps, m = threadIdx.x - kWsGatherWarps * 32;
    const double inv_res = 1.0 / G.L.res;
    CtaRows &R = sh.rows;
    for (int it = 0; it < num_iters; ++it) {
        GnWarpAcc A;
        const bool skip = (P.debug_flags & 2) != 0;
        const int lo = skip ? 0 : c_lo, hi = skip ? 0 : c_hi;
        const bool rigid = P.rigid_first && it == 0;
        RawPoint kr[kWsRowsPerLane];
        const auto load_chunk = [&](int base, int n) {
#pragma unroll
            for (int j = 0; j < kWsRowsPerLane; ++j) {
                const int r = m + j * kWsMathWarps * 32;
                if (r < n) kr[j] = load_raw(keypoints, P.kp_lo, base + r);
            }
        };
        load_chunk(lo, (hi - lo) > kRowCap ? kRowCap : hi - lo);
        if (mw == 0) {
            if (it == 0) {   // the state the host uploaded
                if (lane == 0) {
                    const IcpState *gst = sh.grp.st;
                    const int done = __ldcg(&gst->done);   // issued with the pose loads: one round trip, not two
                    sh.pose = load_pose(gst);
                    sh.done = done;
                }
            } else {
                gn_fetch_pose(sh, tag0 + (unsigned int) it, kLoopSyncTimeout, lane);
            }
            if (lane == 0) R.next = 0;
        }
        gn_ws_math_sync();
        const bool done = sh.done != 0;
        for (int base = lo;; base += kRowCap) {
            const int top = (hi - base) > kRowCap ? base + kRowCap : hi;
            const int n = top > base ? top - base : 0;
            if (!done) {
                if (base != lo) load_chunk(base, n);
#pragma unroll
                for (int j = 0; j < kWsRowsPerLane; ++j) {
                    const int r = m + j * kWsMathWarps * 32;
                    if (r < n) {
                        V3 p;
                        int kx, ky, kz;
                        gn_phase_a(G, kr[j], sh.pose, rigid, inv_res, p, kx, ky, kz);
                        sh.ws.q[r] = WsQuery{p.x, p.y, p.z, kx, ky, kz};
                    }
                }
            }
            sync();   // phase A of the chunk
            if (done) break;
            sync();   // phase B of the chunk
#pragma unroll
            for (int j = 0; j < kWsRowsPerLane; ++j) {
                const int r = m + j * kWsMathWarps * 32;
                if (r < n) {
                    const WsQuery &q = sh.ws.q[r];
                    R.used[r] = gn_phase_c(P, [&] { return kr[j]; }, sh.pose, V3{q.x, q.y, q.z}, need, R.u[r], R.u[r], A) ? 1 : 0;
                }
            }
            gn_store_warp_row(sh.acc[mw], A, lane);   // the counters so far: final after the last chunk
            double unused = 0;   // (no accumulator of the reduction falls on a math warp: kRowParts * kAcc <= gather threads)
            gn_cta_reduce_rows(R, n, unused, sync);
            if (top >= hi) break;
            sync();
        }
        if (done || it == num_iters - 1) break;
    }
}
static_assert(kRowParts * kAcc <= kWsGatherWarps * 32, "the row reduction runs on the gather warps");

// solver CTA, gather warp w: its tagged rows (warps < kGatherWarps) and the sum of the per-warp partials
__device__ __forceinline__ void gn_ws_solver_gather(GnShared &sh, int num_iters, unsigned int tag0, int lane, int w) {
    const GnWsSync sync;
    for (int it = 0; it < num_iters; ++it) {
        if (sh.state.done) break;
        double a0 = 0, a1 = 0, a2 = 0;
        bool ok = true;
        if (w < kGatherWarps) ok = gn_consume_tagged_rows(sh.grp.rows, sh.grp.gather_ctas, tag0 + (unsigned int) it, lane, w, a0, a1, a2);
        if (!gn_ws_sync_and(ok)) break;
        gn_sum_warp_partials(sh, a0, a1, a2, lane, w, sync);
        sync();   // the solve is done with sh.acc / sh.state
    }
}

// solver CTA, math warps: the first one solves, publishes the pose, and after the loop the state and the frame's tail
__device__ __forceinline__ void gn_ws_solver_math(GnShared &sh, int num_iters, unsigned int tag0, FrameTailArgs &tail,
                                                  int lane, int w) {
    const GnWsSync sync;
    const GnParams &P = sh.group.cfg.P;
    const bool solver = w == kWsGatherWarps;
    long long t_loop = 0, t_solve = 0;
    if (solver) {
        if (!(P.debug_flags & 4)) {
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
        t_loop = clock64();
    }
    for (int it = 0; it < num_iters; ++it) {
        const unsigned int tag = tag0 + (unsigned int) it;
        if (sh.state.done) break;
        if (!gn_ws_sync_and(true)) {
            // a gather CTA's row never arrived: give up (the host raises "Error During Optimization"); pose words of
            // the next iteration with done = 1 release every gather CTA that waits for them
            if (solver) {
                if (lane == 0) {
                    sh.state.failed = 2;
                    sh.state.done = 1;
                }
                __syncwarp();
                gn_publish_pose(sh.grp.pose, sh.state, tag + 1u, lane);
            }
            break;
        }
        gn_sum_warp_partials(sh, 0.0, 0.0, 0.0, lane, w, sync);
        if (solver) {
            const long long t_begin = clock64();
            IcpState *ws = &sh.state;
            if (P.debug_flags & 1) {
                if (lane == 0) ws->iter += 1;
            } else
                warp_gn_solve(sh.acc[0], sh.solve, ws, P, 0, nullptr, lane);
            __syncwarp();
            // the gather CTAs wait for the pose words only when they have another iteration to run
            if (it + 1 < num_iters) gn_publish_pose(sh.grp.pose, *ws, tag + 1u, lane);
            if (lane == 0) {
                t_solve += clock64() - t_begin;
                ws->cycles_total = (unsigned long long) (clock64() - t_loop);
                ws->cycles_solve = (unsigned long long) t_solve;
            }
        }
        sync();
    }
    if (!solver) return;
    // the registration's state, published once on every way out of the loop (the host, k_frame_policy and later launches
    // read it after this kernel)
    {
        const int *src = reinterpret_cast<const int *>(&sh.state);
        int *dst = reinterpret_cast<int *>(sh.grp.st);
        for (int i = lane; i < (int) (sizeof(IcpState) / sizeof(int)); i += 32) dst[i] = src[i];
    }
    // ---- the tail of the registration (frame_policy.h): as in k_gn_persistent's other layout
    if (tail.enabled) {
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

// the whole loop of one CTA from the register split on; all kWsWarps warps call
__device__ __forceinline__ void gn_ws_loop(GnShared &sh, const GatherConfig &gather_G, const int *stencil, int num_iters,
                                           bool solver_cta, int c_lo, int c_hi, unsigned int tag0, FrameTailArgs &tail,
                                           int lane, int w) {
    if (w >= kWsGatherWarps) {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kWsMathRegs));
        if (solver_cta) gn_ws_solver_math(sh, num_iters, tag0, tail, lane, w);
        else gn_ws_gather_math(sh, gather_G, num_iters, c_lo, c_hi, tag0, lane, w);
    } else {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kWsGatherRegs));
        if (solver_cta) gn_ws_solver_gather(sh, num_iters, tag0, lane, w);
        else gn_ws_gather_warp(sh, gather_G, stencil, num_iters, c_lo, c_hi, tag0, lane, w);
    }
}

// ---- persistent variant: the WHOLE Gauss-Newton loop in one cooperative launch --------------------------------
// CTA 0 is the solver CTA (deterministic reduction of the partials + 12x12 solve + pose update, by the same warp on
// the same SM every iteration, so its instructions stay in that SM's instruction cache: executed cold, the serial tail
// costs tens of microseconds per iteration, warm a few); CTAs 1..G gather. The two sides meet through the tagged words
// above (-DCTICP_GN_GRID_BARRIERS: two grid-wide barriers per iteration around the same hand-off, the round's earlier
// form). While the gather CTAs work on iteration 0, the solver warp runs the solve once on a dummy system to pull its code
// into the instruction cache. With `tail.enabled` the solver CTA also decides the frame's tail after the loop
// (frame_policy.h).
//
// Groups (kGrouped, GnGroups): one launch runs B independent registrations, each on its own contiguous range of CTAs with
// its own map, options, keypoints, iteration count, solver CTA, state, partial rows and pose words; everything above holds
// per group. A group that converges or fails leaves the loop alone while the others go on, and one group's serial tail
// overlaps the others' gathers. Each CTA copies its group's entry to shared memory and reads it from there; the solo
// instantiation copies its kernel parameters to the same place and never reads the table. kPeers and the frame tail are solo.
//
// kPeers (multi-GPU, keypoints sharded): between its reduction and its solve the solver CTA exchanges the accumulator
// with the other ranks' solver CTAs through NVLink peer memory (peer_exchange.cuh) — the all-reduce of SURVEY §8e
// happens INSIDE the loop, so the sharded loop is still one launch and costs one NVLink round trip per iteration.
template <bool kPeers, bool kGrouped>
__global__ void __launch_bounds__(gn_persistent_threads(kPeers), 1)
k_gn_persistent(GatherLaunch solo_cfg, const float4 *__restrict__ solo_keypoints, const int *__restrict__ d_num_keypoints,
                IcpState *st, int solo_iters, PeerLinks links, GnLoopWords words, FrameTailArgs tail, GnGroups groups) {
    static_assert(!(kPeers && kGrouped), "the sharded loop is single-group");
    constexpr bool kWs = gn_persistent_threads(kPeers) == kWsWarps * 32;   // the warp-specialised loop (gn_ws_loop)
#ifndef CTICP_GN_FLAG_SYNC
    cg::grid_group grid = cg::this_grid();
#endif
    GnShared &sh = *reinterpret_cast<GnShared *>(gn_smem_raw);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    // this CTA's group (GnGroups): from here on the group is the whole registration — `cta` is the index within the
    // group, `group_ctas` its size, and the state / rows / pose words / keypoints are the group's own
    int g = 0, cta = blockIdx.x, group_ctas = gridDim.x;
    unsigned long long *rows = words.rows, *pose_words = words.pose;
    if constexpr (kGrouped) {
        const int *first_cta = groups.first_cta;
        while (first_cta[g + 1] <= (int) blockIdx.x) ++g;
        cta = (int) blockIdx.x - first_cta[g];
        group_ctas = first_cta[g + 1] - first_cta[g];
        rows += (size_t) (first_cta[g] - g) * kRowWords;   // the gather CTAs of the groups before this one
        pose_words += (size_t) kPoseGroupWords * g;
        const int *src = reinterpret_cast<const int *>(groups.table + g);
        int *dst = reinterpret_cast<int *>(&sh.group);
        for (int i = threadIdx.x; i < (int) (sizeof(GnGroup) / sizeof(int)); i += blockDim.x) dst[i] = src[i];
        __syncthreads();
        st = sh.group.st;
    } else {
        // the solo launch keeps its parameters in the same place: read from shared memory where used, they hold no
        // registers across the gather (read from the kernel parameters, some stayed live and `-Xptxas -v` showed 232 / 320 B
        // of spill stores / loads instead of 124 / 176 B)
        if (threadIdx.x == 0) sh.group = GnGroup{solo_cfg, solo_keypoints, d_num_keypoints, st, solo_iters};
        __syncthreads();
    }
    const GatherLaunch &cfg = sh.group.cfg;
    const float4 *__restrict__ keypoints = sh.group.keypoints;
    const GnParams &P = cfg.P;
    // except the gather's map level and radius, which its inner loops read: from the kernel parameters in the solo launch
    // (with every field from shared memory, dense128_gn's wide tiles took 4 % longer)
    const GatherConfig &gather_G = kGrouped ? sh.group.cfg.G : solo_cfg.G;
    const int num_iters = sh.group.num_iters;
    const bool solver_cta = cta == 0;
    unsigned int peer_seq = 0;   // sequence number of the last exchange (solver CTA only)
    if (kPeers && solver_cta) peer_seq = *links.seq;
    const int gather_ctas = group_ctas - 1;
    const int *stencil = stencil_table_fill(sh.stencil, cfg.G.r);
    if (threadIdx.x == 0) {
        sh.grp.st = st;
        sh.grp.rows = solver_cta ? rows : rows + (size_t) (cta - 1) * kRowWords;
        sh.grp.pose = pose_words;
        sh.grp.gather_ctas = gather_ctas;
    }
    for (int i = threadIdx.x; i < kRowCap; i += blockDim.x) sh.rows.cost[i] = 0u;   // iteration 0's paired schedule
    __syncthreads();

    if (solver_cta) {   // working copy of the state in shared memory: the serial tail never waits for global memory
        const int *src = reinterpret_cast<const int *>(st);
        int *dst = reinterpret_cast<int *>(&sh.state);
        for (int i = threadIdx.x; i < (int) (sizeof(IcpState) / sizeof(int)); i += blockDim.x) dst[i] = src[i];
        __syncthreads();
    }
    CT_STAMP(if (solver_cta && threadIdx.x < 4) sh.state.dbg_t[threadIdx.x] = 0; __syncthreads();)
    if (!kWs && solver_cta && w == 0 && !(P.debug_flags & 4)) {
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
    if (!kWs) {
        sel_bulk_init(bulk, &sh.mbar[w], lane);
        bulk_ptr = &bulk;
    }
#endif
    long long t_loop = 0, t_solve = 0;
    if (solver_cta && threadIdx.x == 0) t_loop = clock64();
    // this rank's keypoint range and the tile width: constant over the iterations (integer divisions)
    const int K = *sh.group.num_keypoints;
    int kp_lo = 0, kp_hi = K;
    if (P.shard_world > 1) {
        kp_lo = (int) ((long long) K * P.shard_rank / P.shard_world);
        kp_hi = (int) ((long long) K * (P.shard_rank + 1) / P.shard_world);
    }
    // this CTA's balanced share of the range
    int c_lo = 0, c_hi = 0;
    if (!solver_cta) {
        c_lo = kp_lo + (int) ((long long) (kp_hi - kp_lo) * (cta - 1) / gather_ctas);
        c_hi = kp_lo + (int) ((long long) (kp_hi - kp_lo) * cta / gather_ctas);
    }
    if constexpr (kWs) {
        gn_ws_loop(sh, gather_G, stencil, num_iters, solver_cta, c_lo, c_hi, words.tag, tail, lane, w);
        return;
    }
    for (int it = 0; it < num_iters; ++it) {
        const unsigned int tag = words.tag + (unsigned int) it;
        if (solver_cta) {
            if (sh.state.done) break;
        } else {
            GnWarpAcc A;
            CT_STAMP(const long long t_it = clock64();)
            // a range of more keypoints than warps but at most two per warp takes the paired schedule, built from the last
            // iteration's costs by warp 1 while warp 0 waits for the pose; the first iteration has no costs yet (all zero:
            // the schedule in keypoint order). With CTICP_DEBUG_FLAGS & 8, a debug switch for bit-identity tests, every
            // iteration takes tiles of one keypoint grabbed from the counter.
            const bool paired = !(P.debug_flags & (2 | 8)) && gn_pairs_apply(c_hi - c_lo);
            if (w == 1 && paired) gn_pair_schedule(sh.rows, c_hi - c_lo, lane);
            if (w == 0) {   // phases A / C read the pose from shared memory: 34 registers less to keep live
                if (it == 0) {   // the state the host uploaded
                    if (lane == 0) {
                        const IcpState *gst = sh.grp.st;
                        const int done = __ldcg(&gst->done);   // issued with the pose loads: one round trip, not two
                        sh.pose = load_pose(gst);
                        sh.done = done;
                    }
                } else {
                    // (sharded: the solver CTA may itself be waiting for a late peer rank, up to PeerLinks::timeout_cycles)
                    gn_fetch_pose(sh, tag, kLoopSyncTimeout + (kPeers ? links.timeout_cycles : 0LL), lane);
                }
                if (lane == 0) sh.rows.next = 0;
            }
            __syncthreads();
            if (sh.done) break;
            CT_STAMP(const long long t_g0 = clock64();)
            // (CTICP_DEBUG_FLAGS & 2, timing only: an empty range — the hand-off and the reduction without the gather work)
            const bool skip = (P.debug_flags & 2) != 0;
            const double s = gn_cta_gather(gather_G, P, stencil, keypoints, skip ? 0 : c_lo, skip ? 0 : c_hi, sh, lane, w, A, bulk_ptr,
                                           P.rigid_first && it == 0, paired);
            if (threadIdx.x < kAcc) tagged_store_double(sh.grp.rows + 2 * threadIdx.x, tag, s);
            CT_STAMP(const long long t_g = clock64();)
            CT_STAMP(const int dbg_kp = __reduce_add_sync(0xffffffffu, A.n_kp);)
            CT_STAMP(if (P.dbg_warp && lane == 0 && it < kDbgIters) {
                unsigned long long *o = P.dbg_warp + ((size_t) it * (gather_ctas * kGatherWarps) + (w * gather_ctas + (cta - 1))) * kDbgSlots;
                o[0] = (unsigned long long) A.dbg[0]; o[1] = (unsigned long long) A.dbg[1];
                o[2] = (unsigned long long) A.dbg[2];
                o[3] = (unsigned long long) (t_g0 - t_it);         // pose fetch + barrier
                o[4] = (unsigned long long) (t_g - t_it);          // pose fetch + tiles + CTA row reduction
                o[5] = 0;
                o[6] = A.dbg[3] ? (unsigned long long) (A.dbg[3] - t_g0) : 0;   // end of the warp's last tile
                o[7] = (unsigned long long) dbg_kp | ((unsigned long long) A.dbg[4] << 8);   // keypoints | longest tile << 8
            })
#ifdef CTICP_GN_FLAG_SYNC
            if (it == num_iters - 1) break;   // nothing left to wait for: the solver CTA finishes the registration alone
#endif
        }
        CT_STAMP(const long long t_bar = clock64();)
#ifndef CTICP_GN_FLAG_SYNC
        grid.sync();
#endif
        CT_STAMP(if (!solver_cta && P.dbg_warp && lane == 0 && w == 0 && it < kDbgIters) {
            // (slot 5 of this CTA's first warp is overwritten with the wait at the barrier that follows the gather)
            unsigned long long *o = P.dbg_warp + ((size_t) it * (gather_ctas * kGatherWarps) + (cta - 1)) * kDbgSlots;
            o[5] = (unsigned long long) (clock64() - t_bar);
        })
        if (solver_cta) {
            CT_STAMP(const long long t_red = clock64();)
            if (!gn_reduce_tagged_rows(sh, sh.grp.rows, sh.grp.gather_ctas, tag, lane, w)) {
                // a gather CTA's row never arrived: give up (the host raises "Error During Optimization"); pose words of
                // the next iteration with done = 1 release every gather CTA that waits for them
                if (w == 0) {
                    if (lane == 0) {
                        sh.state.failed = 2;
                        sh.state.done = 1;
                    }
                    __syncwarp();
                    gn_publish_pose(sh.grp.pose, sh.state, tag + 1u, lane);
                }
                break;
            }
            // -DCTICP_DEBUG_TIMERS: SM cycles summed over the iterations — dbg_t[0] reduction of the partial rows,
            // [1] everything from there to the published pose, [2] the 12x12 solve, [3] the pose update
            const long long t_begin = threadIdx.x == 0 ? clock64() : 0;
            CT_STAMP(if (threadIdx.x == 0) sh.state.dbg_t[0] += (unsigned long long) (t_begin - t_red);)
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
                // the gather CTAs wait for the pose words only when they have another iteration to run
                if (it + 1 < num_iters) gn_publish_pose(sh.grp.pose, *ws, tag + 1u, lane);
                if (lane == 0) {
                    t_solve += clock64() - t_begin;
                    ws->cycles_total = (unsigned long long) (clock64() - t_loop);
                    ws->cycles_solve = (unsigned long long) t_solve;
                }
                CT_STAMP(if (lane == 0) ws->dbg_t[1] += (unsigned long long) (clock64() - t_rest);)
            }
            __syncthreads();   // warp 0 is done with sh.acc / sh.state before the next iteration's reduction
        }
#ifndef CTICP_GN_FLAG_SYNC
        grid.sync();
#endif
    }
    if (kPeers && solver_cta && threadIdx.x == 0) *links.seq = peer_seq;
    if (!solver_cta) return;
    __syncthreads();   // sh.state is final
    if (w != 0) return;
    // the registration's state, published once on every way out of the loop (the host, k_frame_policy and later launches
    // read it after this kernel)
    {
        const int *src = reinterpret_cast<const int *>(&sh.state);
        int *dst = reinterpret_cast<int *>(sh.grp.st);
        for (int i = lane; i < (int) (sizeof(IcpState) / sizeof(int)); i += 32) dst[i] = src[i];
    }
    // ---- the tail of the registration (frame_policy.h): AssessRegistration + the insertion policy on the final state, the
    // verdict to HBM (the speculative map update launched behind this kernel reads it) and to mapped pinned host memory
    if (tail.enabled) {
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
    cudaFuncGetAttributes(&a, k_gn_persistent<true, false>);
    cudaFuncGetAttributes(&a, k_gn_persistent<false, false>);
    cudaFuncGetAttributes(&a, k_gn_iterate);
    cudaFuncGetAttributes(&a, k_peer_allreduce);
    cudaFuncGetAttributes(&a, k_gn_solve_acc);
    PreloadLmKernels();
    cudaGetLastError();
}
void IcpSolver::AllReduceAccumulator(void *nccl_comm, IcpState *d_state) {
    if (peers_ready_) {
        k_peer_allreduce<<<1, 256, 0, stream_>>>(PeerLinksOf(links_host_), d_acc_.data(), d_state);
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
    CT_CUDA_CHECK(cudaFuncSetAttribute(k_gn_persistent<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) sizeof(GnShared)));
    CT_CUDA_CHECK(cudaFuncSetAttribute(k_gn_persistent<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) sizeof(GnShared)));
    CT_CUDA_CHECK(cudaFuncSetAttribute(k_gn_persistent<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) sizeof(GnShared)));
    cudaDeviceGetAttribute(&num_sms_, cudaDevAttrMultiProcessorCount, dev);
    d_sys_.reserve(160, stream_);
    d_acc_.reserve(kAcc, stream_);
    d_ticket_.reserve(1, stream_);
    CT_CUDA_CHECK(cudaMemset(d_ticket_.data(), 0, sizeof(unsigned int)));
    for (int i = 0; i < kMaxEvents; ++i) {
        ev_begin_[i] = Event(cudaEventDefault);
        ev_end_[i] = Event(cudaEventDefault);
    }
}
void IcpSolver::EnsurePartials(int blocks) { d_partials_.reserve((size_t) kAcc * blocks, stream_); }
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
int IcpSolver::GnCoresident(bool peers) {
    int &coresident = max_coresident_[peers ? 1 : 0];
    if (coresident == 0) {
        void *kernel = peers ? (void *) k_gn_persistent<true, false> : (void *) k_gn_persistent<false, false>;
        int per_sm = 0;
        CT_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, gn_persistent_threads(peers), sizeof(GnShared)));
        coresident = std::max(1, per_sm * num_sms_);
    }
    return coresident;
}

// The words of the persistent loop (GnLoopWords) for `rows` gather CTAs and `groups` groups, grown on demand and zeroed when
// allocated, and the tag of iteration 0 of a launch of `num_iters` iterations: the counter advances by num_iters + 1 per
// launch. Tag 0 is never handed out, so zeroed words never match; when the counter would wrap, both areas are zeroed
// again (stream order: after every earlier launch) and it restarts at 1.
unsigned int IcpSolver::ReserveLoopTags(int rows, int groups, int num_iters) {
    const auto grow = [&](DeviceArray<unsigned long long> &buf, size_t words) {
        if (words <= buf.capacity()) return;
        buf.reserve(words, stream_);
        CT_CUDA_CHECK(cudaMemsetAsync(buf.data(), 0, sizeof(unsigned long long) * words, stream_));
    };
    grow(d_loop_rows_, kRowWords * (size_t) std::max(rows, 1));
    grow(d_loop_pose_, kPoseGroupWords * (size_t) std::max(groups, 1));
    const unsigned long long span = (unsigned long long) std::max(num_iters, 0) + 1;
    if (loop_tag_ + span > 0xffffffffull) {
        CT_CUDA_CHECK(cudaMemsetAsync(d_loop_rows_.data(), 0, sizeof(unsigned long long) * d_loop_rows_.capacity(), stream_));
        CT_CUDA_CHECK(cudaMemsetAsync(d_loop_pose_.data(), 0, sizeof(unsigned long long) * d_loop_pose_.capacity(), stream_));
        loop_tag_ = 1;
    }
    const unsigned int tag = loop_tag_;
    loop_tag_ += (unsigned int) span;
    return tag;
}

bool IcpSolver::batch_supported() const {
#ifdef CTICP_GN_FLAG_SYNC
    return use_persistent_;
#else
    return false;
#endif
}

void IcpSolver::EnqueueGaussNewtonBatch(const DeviceMap &map, const cticp_icp_options &opt, int batch, const size_t *h_n,
                                        const float4 *d_keypoints, int num_iters, IcpState *d_states) {
    if (batch < 1) throw std::invalid_argument("batch must be at least 1");
    std::vector<GnProblem> problems(batch);
    size_t base = 0;
    for (int b = 0; b < batch; ++b) {
        problems[b] = GnProblem{&map, &opt, d_keypoints + base, kp_lo_ ? kp_lo_ + base : nullptr, nullptr, h_n[b], num_iters,
                                d_states + b};
        base += h_n[b];
    }
    EnqueueGaussNewtonGroups(problems.data(), batch);
}

void IcpSolver::EnqueueGaussNewtonGroups(const GnProblem *problems, int batch) {
    if (!batch_supported()) throw std::logic_error("batched Gauss-Newton needs the persistent flag-synchronised loop");
    if (batch < 1) throw std::invalid_argument("batch must be at least 1");
    for (int b = 0; b < batch; ++b)
        if (problems[b].opt->max_number_neighbors > 32 || problems[b].opt->max_number_neighbors < 1)
            throw std::invalid_argument("max_number_neighbors must be in [1, 32]");
    // (k_gn_persistent<false, true> has the launch bounds and the shared memory of the solo kernel: the same occupancy)
    const int coresident = GnCoresident(false);
    if (2 * batch > coresident)
        throw CapacityError("batch of " + std::to_string(batch) + " registrations: the device holds " +
                                std::to_string(coresident) + " CTAs of the Gauss-Newton kernel, two per registration needed");
    // table: GnGroup[B] | first_cta[0..B] | the counts of the problems without a device count
    std::vector<size_t> n(batch);
    for (int b = 0; b < batch; ++b) n[b] = problems[b].n;
    std::vector<int> gather(batch);
    BatchGatherCtas(n.data(), batch, coresident, kp_per_cta_, gather.data());
    const size_t cta_off = sizeof(GnGroup) * (size_t) batch, count_off = cta_off + sizeof(int) * (size_t) (batch + 1);
    const size_t bytes = count_off + sizeof(int) * (size_t) batch;
    d_gn_table_.reserve(bytes, stream_);
    h_gn_table_.assign(bytes, 0);
    GnGroup *table = reinterpret_cast<GnGroup *>(h_gn_table_.data());
    int *first_cta = reinterpret_cast<int *>(h_gn_table_.data() + cta_off);
    int *count = reinterpret_cast<int *>(h_gn_table_.data() + count_off);
    const int *d_count = reinterpret_cast<const int *>(d_gn_table_.data() + count_off);
    int max_iters = 0;
    for (int b = 0; b < batch; ++b) {
        const GnProblem &p = problems[b];
        if (p.n > (size_t) INT32_MAX) throw std::invalid_argument("too many keypoints in one problem");
        GnGroup &e = table[b];
        e.cfg.P = MakeParams(*p.map, *p.opt);
        e.cfg.P.kp_lo = p.keypoints_lo;
        e.cfg.G.L = p.map->Level(e.cfg.P.level);
        e.cfg.G.r = e.cfg.P.r;
        e.cfg.G.radius2 = e.cfg.P.radius * e.cfg.P.radius;
        e.cfg.G.kmax = e.cfg.P.kmax;
        e.keypoints = p.keypoints;
        count[b] = (int) p.n;
        e.num_keypoints = p.d_num_keypoints ? p.d_num_keypoints : d_count + b;
        e.st = p.d_state;
        e.num_iters = p.num_iters;
        max_iters = std::max(max_iters, p.num_iters);
        first_cta[b + 1] = first_cta[b] + 1 + gather[b];
    }
    const int grid = first_cta[batch];
    CT_CUDA_CHECK(cudaMemcpyAsync(d_gn_table_.data(), h_gn_table_.data(), bytes, cudaMemcpyHostToDevice, stream_));
    const unsigned int tag = ReserveLoopTags(grid - batch, batch, max_iters);
    GnLoopWords words{d_loop_rows_.data(), d_loop_pose_.data(), tag};
    GatherLaunch cfg{};
    const float4 *kp = nullptr;
    const int *nk = nullptr;
    IcpState *st = nullptr;
    int iters = 0;
    PeerLinks links{};
    FrameTailArgs tail_args{};
    GnGroups groups{reinterpret_cast<const GnGroup *>(d_gn_table_.data()), reinterpret_cast<const int *>(d_gn_table_.data() + cta_off), batch};
    void *args[] = {&cfg, &kp, &nk, &st, &iters, &links, &words, &tail_args, &groups};
    CT_CUDA_CHECK(cudaLaunchCooperativeKernel((void *) k_gn_persistent<false, true>, dim3(grid), dim3(gn_persistent_threads(false)), args,
                                              sizeof(GnShared), stream_));
    gather_launches_ += 1;
    launches_ += 1;
}

void IcpSolver::PrintWarpStamps(int iters) {
#ifdef CTICP_DEBUG_TIMERS
    if (!d_dbg_warp_.data() || dbg_warps_ <= 0) return;
    const int W = dbg_warps_;
    std::vector<unsigned long long> h((size_t) kDbgIters * W * kDbgSlots);
    CT_CUDA_CHECK(cudaMemcpy(h.data(), d_dbg_warp_.data(), sizeof(unsigned long long) * h.size(), cudaMemcpyDeviceToHost));
    static const char *names[kDbgSlots - 1] = {"A pose+voxel", "B gather+select", "C epilogue", "pose fetch", "fetch+tiles+row reduction",
                                               "barrier wait (per CTA)", "end of last tile"};
    const auto pct = [](std::vector<unsigned long long> v, int p) { std::sort(v.begin(), v.end()); return v.empty() ? 0ull : v[v.size() * p / 100]; };
    for (int it = 0; it < std::min(iters, kDbgIters); ++it) {
        const unsigned long long *h_it = h.data() + (size_t) it * W * kDbgSlots;
        // per CTA: the warp whose last tile ends last, the keypoints it took, the CTA's longest single tile
        const int ctas = W / kGatherWarps;
        int last_two = 0, ctas_seen = 0, slowest_cta = -1;
        unsigned long long slowest_end = 0, a = 0, b = 0, c = 0, kps = 0;
        std::vector<unsigned long long> cta_end, cta_tile, excess;
        for (int ct = 0; ct < ctas; ++ct) {
            unsigned long long end = 0, tile = 0;
            int last_kp = 0;
            for (int w = 0; w < kGatherWarps; ++w) {
                const unsigned long long *o = h_it + ((size_t) w * ctas + ct) * kDbgSlots;
                if (o[4] == 0) continue;
                a += o[0]; b += o[1]; c += o[2]; kps += o[7] & 0xff;
                tile = std::max(tile, o[7] >> 8);
                if (o[6] >= end) { end = o[6]; last_kp = (int) (o[7] & 0xff); }
            }
            if (end == 0) continue;
            ++ctas_seen;
            last_two += last_kp >= 2;
            cta_end.push_back(end);
            cta_tile.push_back(tile);
            excess.push_back(end > tile ? end - tile : 0);
            if (end > slowest_end) { slowest_end = end; slowest_cta = last_kp; }
        }
        if (ctas_seen > 0 && kps > 0)
            fprintf(stderr, "[cticp] GN gather CTAs, iteration %d: %d CTAs; last warp held >= 2 keypoints in %d; slowest CTA %llu "
                    "(its last warp %d keypoints); CTA tiles end p50 %llu p90 %llu; longest single tile p50 %llu p90 %llu; "
                    "end - longest tile p50 %llu p90 %llu; per keypoint A %.0f B %.0f C %.0f\n", it, ctas_seen, last_two,
                    slowest_end, slowest_cta, pct(cta_end, 50), pct(cta_end, 90), pct(cta_tile, 50), pct(cta_tile, 90),
                    pct(excess, 50), pct(excess, 90), (double) a / kps, (double) b / kps, (double) c / kps);
        fprintf(stderr, "[cticp] GN gather warps, iteration %d (SM cycles; %d warps):", it, W);
        for (int sl = 0; sl < kDbgSlots - 1; ++sl) {
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
        cudaEventSynchronize(ev_end_[i].get());
        if (cudaEventElapsedTime(&ms, ev_begin_[i].get(), ev_end_[i].get()) == cudaSuccess) gather_ms_ += ms;
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
        void *kernel = peers ? (void *) k_gn_persistent<true, false> : (void *) k_gn_persistent<false, false>;
        const int coresident = GnCoresident(peers);
        const int blocks = GatherBlocks(k_share, std::max(1, coresident - 1), kp_per_cta_);
        int grid = std::min(blocks + 1, coresident);
        grid = std::max(grid, 2);
        const float4 *kp = d_keypoints;
        const int *nk = d_num_keypoints;
        int iters = num_iters;
        PeerLinks links = peers ? PeerLinksOf(links_host_) : PeerLinks{};
#ifdef CTICP_DEBUG_TIMERS
        if (getenv("CTICP_DEBUG_TIMERS")) {
            const int warps = (grid - 1) * kGatherWarps;
            d_dbg_warp_.reserve((size_t) kDbgIters * warps * kDbgSlots, stream_);
            dbg_warps_ = warps;
            CT_CUDA_CHECK(cudaMemsetAsync(d_dbg_warp_.data(), 0, sizeof(unsigned long long) * kDbgIters * warps * kDbgSlots, stream_));
            cfg.P.dbg_warp = d_dbg_warp_.data();
        }
#endif
        const unsigned int tag = ReserveLoopTags(grid - 1, 1, num_iters);
        GnLoopWords words{d_loop_rows_.data(), d_loop_pose_.data(), tag};
        FrameTailArgs tail_args{};
        if (tail) tail_args = *tail;
        GnGroups groups{nullptr, nullptr, 1};
        void *args[] = {&cfg, &kp, &nk, &d_state, &iters, &links, &words, &tail_args, &groups};
        const bool timed = time_gather_ && ev_used_ < kMaxEvents;
        if (timed) cudaEventRecord(ev_begin_[ev_used_].get(), stream_);
        CT_CUDA_CHECK(cudaLaunchCooperativeKernel(kernel, dim3(grid), dim3(gn_persistent_threads(peers)), args, sizeof(GnShared), stream_));
        if (timed) cudaEventRecord(ev_end_[ev_used_++].get(), stream_);
        gather_launches_ += 1;
        launches_ += 1;
        return tail != nullptr;
    }
    const int blocks = GatherBlocks(k_share, num_sms_, kp_per_cta_);
    EnsurePartials(blocks + 1);
    for (int it = 0; it < num_iters; ++it) {
        const bool timed = time_gather_ && ev_used_ < kMaxEvents;
        if (timed) cudaEventRecord(ev_begin_[ev_used_].get(), stream_);
        k_gn_iterate<<<blocks, kGatherWarps * 32, sizeof(GnShared), stream_>>>(cfg, d_keypoints, d_num_keypoints, d_state,
                                                                              d_partials_.data(), d_ticket_.data(), nccl_comm ? 2 : 0, d_acc_.data(), nullptr);
        if (timed) cudaEventRecord(ev_end_[ev_used_++].get(), stream_);
        ++gather_launches_;
        launches_ += 1;
        if (nccl_comm) {
            AllReduceAccumulator(nccl_comm, d_state);   // in-place sum of d_acc_ over ranks (peer mailboxes, else NCCL)
            k_gn_solve_acc<<<1, 32, 0, stream_>>>(d_acc_.data(), d_state, cfg.P);
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
    CT_CUDA_CHECK(cudaMemsetAsync(d_sys_.data(), 0, sizeof(double) * 160, stream_));
    k_gn_iterate<<<blocks, kGatherWarps * 32, sizeof(GnShared), stream_>>>(cfg, d_keypoints, d_num_keypoints, d_state,
                                                                          d_partials_.data(), d_ticket_.data(), 1, d_acc_.data(), d_sys_.data());
    launches_ += 1;
    double h[160];
    CT_CUDA_CHECK(cudaMemcpyAsync(h, d_sys_.data(), sizeof(h), cudaMemcpyDeviceToHost, stream_));
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
    DeviceArray<RadiusSearchLevels> d_R;
    d_R.reserve(1, stream_);
    CT_CUDA_CHECK(cudaMemcpyAsync(d_R.data(), &R, sizeof(R), cudaMemcpyHostToDevice, stream_));
    const int blocks = (int) std::max<size_t>(1, std::min((n + kGatherWarps - 1) / kGatherWarps, (size_t) num_sms_ * 2));
    k_radius_search<<<blocks, kGatherWarps * 32, 0, stream_>>>(d_R.data(), kmax, d_queries, d_radiuses, (int) n, d_out_points, d_out_counts);
    launches_ += 1;
    CT_CUDA_CHECK(cudaGetLastError());
    CT_CUDA_CHECK(cudaStreamSynchronize(stream_));
}

}  // namespace cticp
