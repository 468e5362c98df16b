// small_solve.cuh — pieces shared by the GN and LM solver kernels: the (i,j) pair table of the packed 12x12 upper
// triangle and the warp-resident 12x12 SPD solve. Each translation unit that includes this header owns a copy of the
// __constant__ tables (statically initialised, see below).
#pragma once
#include <cuda_runtime.h>

#include "icp.h"

namespace cticp {

// (i,j) of the idx-th entry of the row-major upper triangle of a 12x12 matrix; entries 78..89 pair (i, 12).
// Statically initialised: __constant__ memory is per device and per module load, so every device that runs these kernels
// gets the tables with the module — no upload call that could be skipped for a second GPU in the same process.
static __constant__ unsigned char c_pair_i[kAccUsed] = {
    0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2,
    2, 2, 2, 3, 3, 3, 3, 3, 3, 3, 3, 3, 4, 4, 4, 4, 4, 4, 4, 4, 5, 5, 5, 5, 5, 5, 5, 6, 6, 6,
    6, 6, 6, 7, 7, 7, 7, 7, 8, 8, 8, 8, 9, 9, 9, 10, 10, 11, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
static __constant__ unsigned char c_pair_j[kAccUsed] = {
    0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 2, 3, 4, 5, 6, 7, 8,
    9, 10, 11, 3, 4, 5, 6, 7, 8, 9, 10, 11, 4, 5, 6, 7, 8, 9, 10, 11, 5, 6, 7, 8, 9, 10, 11, 6, 7, 8,
    9, 10, 11, 7, 8, 9, 10, 11, 8, 9, 10, 11, 9, 10, 11, 10, 11, 11, 12, 12, 12, 12, 12, 12, 12, 12, 12, 12, 12, 12};

// ---- 12x12 SPD solve by one warp ---------------------------------------------------------------------------
struct SolveScratch {
    double A[12][13];
    double b[12], x[12], D[12], y[12];
    double sn[8], cs[8];
    int perm[12];
};

// Solve the 12x12 SPD system held in S.A / S.b; x → S.x.
// Eigen's A.ldlt().solve(b) (ct_icp.cpp:914) is replaced by Gauss-Jordan elimination in natural order on the augmented
// matrix [A | b] (no back-substitution). The system is symmetric positive definite (JTJ/n plus the diagonal regularisers),
// for which elimination without pivoting is backward stable; the result agrees with a pivoted LDL^T to ~1e-13 relative.
// History of the serial tail this sits in: round 1 kept rows in registers but broadcast all 13 columns at every step and
// back-substituted (~3.5k instructions); the first round-2 form updated the matrix in shared memory (5 entries per lane and
// pivot, two barriers per pivot: ~0.5k instructions but a long serial chain — every pivot waits for a store -> barrier ->
// load round trip); this one is ~0.5k instructions with only shuffle latency between pivots.
static __device__ __forceinline__ void warp_ldlt_solve12(SolveScratch &S, int lane) {
    // Gauss-Jordan on the augmented 12 x 13 system, IN REGISTERS: lane r holds row r; step p broadcasts the pivot row's
    // remaining entries by shuffles, every lane forms the reciprocal of the pivot itself, and each row is updated with
    // fully unrolled, compile-time column indices. (The shared-memory form before it paid two barriers plus a
    // store -> load round trip per pivot.) Same operations on the
    // same operands as before: the pivot row is scaled by 1 / pivot, row r loses (a_rp / pivot) x the OLD pivot row.
    const int r = lane < 12 ? lane : 0;   // lanes 12..31 mirror row 0 (their results are discarded)
    double a[13];
#pragma unroll
    for (int c = 0; c < 12; ++c) a[c] = S.A[r][c];
    a[12] = S.b[r];
#pragma unroll
    for (int p = 0; p < 12; ++p) {
        const double pd = __shfl_sync(0xffffffffu, a[p], p);
        const double inv = (fabs(pd) > 2.2250738585072014e-308) ? 1.0 / pd : 0.0;   // pseudo-inverse like Eigen's D
        const bool is_p = lane == p;
        const double f = a[p] * inv;
#pragma unroll
        for (int c = p + 1; c < 13; ++c) {
            const double apc = __shfl_sync(0xffffffffu, a[c], p);
            a[c] = is_p ? apc * inv : a[c] - f * apc;
        }
    }
    if (lane < 12) S.x[lane] = a[12];
    __syncwarp();
}

// The same elimination on the augmented matrix in shared memory, as a 12-trip loop (five entries per lane and pivot): ~60
// instructions of code instead of ~500. For callers whose serial tail is bound by INSTRUCTION FETCH rather than latency —
// the CERES minimizer step runs ~1k instructions once per evaluation on one warp, cold in the 32 KB L1.5 I-cache every time
// (the workers' code streams through the cache in between): this form measured faster per step than the unrolled
// register form above, inlined or as a call.
static __device__ __forceinline__ void warp_ldlt_solve12_compact(SolveScratch &S, int lane) {
    if (lane < 12) S.A[lane][12] = S.b[lane];   // augmented column
    int er[5], ec[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        const int e = lane + 32 * k;            // 156 entries: rows of 13
        er[k] = e < 156 ? e / 13 : 0;
        ec[k] = e < 156 ? e % 13 : 0;
    }
    __syncwarp();
#pragma unroll 1
    for (int p = 0; p < 12; ++p) {
        const double pd = S.A[p][p];
        const double inv = (fabs(pd) > 2.2250738585072014e-308) ? 1.0 / pd : 0.0;   // pseudo-inverse like Eigen's D
        double nv[5];
#pragma unroll
        for (int k = 0; k < 5; ++k) {
            const double arc = S.A[er[k]][ec[k]], arp = S.A[er[k]][p], apc = S.A[p][ec[k]];
            const double f = arp * inv;
            nv[k] = er[k] == p ? apc * inv : arc - f * apc;
        }
        __syncwarp();   // every lane has read the old matrix
#pragma unroll
        for (int k = 0; k < 5; ++k)
            if (lane + 32 * k < 156) S.A[er[k]][ec[k]] = nv[k];
        __syncwarp();
    }
    if (lane < 12) S.x[lane] = S.A[lane][12];
    __syncwarp();
}


}  // namespace cticp
