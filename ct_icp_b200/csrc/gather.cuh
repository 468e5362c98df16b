// gather.cuh — warp-cooperative neighbor gather for one query point (the hot inner loop).
//
// Replaces MultipleResolutionVoxelMap::RadiusSearchInPlace (include/ct_icp/map.h:449-514, called through
// ComputeNeighborhoodInPlace :527-530 with sensor_location == nullptr) and TNeighborhood::ComputeNeighborhood +
// ComputeNeighborhoodInfo (include/SlamCore/experimental/neighborhood.h:226-257, 286-316).
//
// One warp per query:
//   * lanes probe the (2r+1)^3 stencil voxels in parallel (one 16-byte slot load each, x→y→z order like :470-472);
//   * every occupied voxel's points are read as one coalesced run of float4 (<= B*16 bytes);
//   * distances are evaluated in fp64 from the fp32 voxel-local offsets; in-radius candidates are compacted into a
//     64-entry shared-memory staging buffer by ballot/popc;
//   * the k nearest are kept in a register-resident sorted list (one entry per lane) maintained with a bitonic
//     sort/merge network over warp shuffles; ties resolve to the earlier-scanned point (strict `<` at :495).
// Lane l ends with the l-th nearest neighbor; the reference's points[0] (the FARTHEST kept, :508-513) is lane n-1.
#pragma once
#include "device_map.cuh"

namespace cticp {

struct KnnEntry {
    double d2;        // squared distance (fp64)
    int seq;          // scan order: stencil index * 64 + index in voxel
    uint32_t addr;    // index into MapLevel::points
};

struct __align__(16) KnnStage {
    double d2;
    int seq;
    uint32_t addr;
};

constexpr double kKnnInf = 1e300;

__device__ __forceinline__ bool knn_less(const KnnEntry &a, const KnnEntry &b) {
    // predicate logic only (| and &, not || and &&): the short-circuit form compiled to a divergent branch with a
    // reconvergence barrier in every step of the compare-exchange network, which made the GN loop slower
    const bool lt = a.d2 < b.d2, eq = a.d2 == b.d2, sl = a.seq < b.seq;
    return lt | (eq & sl);
}
__device__ __forceinline__ KnnEntry knn_shfl_xor(const KnnEntry &e, int mask) {
    KnnEntry o;
    o.d2 = __shfl_xor_sync(0xffffffffu, e.d2, mask);
    o.seq = __shfl_xor_sync(0xffffffffu, e.seq, mask);
    o.addr = __shfl_xor_sync(0xffffffffu, e.addr, mask);
    return o;
}
__device__ __forceinline__ void knn_cmpx(KnnEntry &e, int lane, int j, bool keep_min) {
    const KnnEntry o = knn_shfl_xor(e, j);
    const bool o_less = knn_less(o, e);
    if (o_less == keep_min) e = o;
}
// full bitonic sort of 32 entries (one per lane), ascending by (d2, seq)
__device__ __forceinline__ void knn_sort32(KnnEntry &e, int lane) {
#pragma unroll
    for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
        for (int j = k >> 1; j > 0; j >>= 1) {
            const bool up = ((lane & k) == 0) || (k == 32);
            const bool lower = ((lane & j) == 0);
            knn_cmpx(e, lane, j, lower == up);
        }
    }
}
// best (ascending) ← 32 smallest of best ∪ chunk (chunk ascending)
__device__ __forceinline__ void knn_merge32(KnnEntry &best, const KnnEntry &chunk, int lane) {
    KnnEntry rev;
    rev.d2 = __shfl_sync(0xffffffffu, chunk.d2, 31 - lane);
    rev.seq = __shfl_sync(0xffffffffu, chunk.seq, 31 - lane);
    rev.addr = __shfl_sync(0xffffffffu, chunk.addr, 31 - lane);
    if (knn_less(rev, best)) best = rev;   // bitonic sequence holding the 32 smallest
#pragma unroll
    for (int j = 16; j > 0; j >>= 1) knn_cmpx(best, lane, j, (lane & j) == 0);
}

struct GatherConfig {
    MapLevel L;
    int r;              // voxel_neighborhood (stencil radius in voxels)
    double radius2;     // search radius squared
    int kmax;           // max_number_neighbors (<= 32)
};

// stencil index → voxel offset, x outermost / z innermost (map.h:470-472)
__device__ __forceinline__ void stencil_offset(int s, int r, int &dx, int &dy, int &dz) {
    const int side = 2 * r + 1;
    dx = s / (side * side) - r;
    dy = (s / side) % side - r;
    dz = s % side - r;
}
// The (2r+1)^3 offsets are tabulated once per CTA in shared memory (packed dx+r | dy+r << 8 | dz+r << 16):
// the integer divisions above were 14% of the kernel's instructions when evaluated per voxel visit.
constexpr int kMaxStencil = 729;   // r <= 4
// Returns the table, or nullptr when the stencil is too large to tabulate (r > 4: offsets are then computed on the
// fly — correct for any radius, e.g. the reference's own map test uses voxel 0.01 with radius 0.8).
__device__ __forceinline__ const int *stencil_table_fill(int *table, int r) {
    const int side = 2 * r + 1, nst = side * side * side;
    if (r > 4) return nullptr;
    for (int s = threadIdx.x; s < nst; s += blockDim.x) {
        int dx, dy, dz;
        stencil_offset(s, r, dx, dy, dz);
        table[s] = (dx + r) | ((dy + r) << 8) | ((dz + r) << 16);
    }
    return table;
}
__device__ __forceinline__ void stencil_lookup(const int *table, int s, int r, int &dx, int &dy, int &dz) {
    if (table) {
        const int packed = table[s];
        dx = (packed & 0xff) - r;
        dy = ((packed >> 8) & 0xff) - r;
        dz = ((packed >> 16) & 0xff) - r;
    } else {
        stencil_offset(s, r, dx, dy, dz);
    }
}

// query point and its voxel (slam::Voxel::Coordinates: three fp64 divisions, done once, one per lane 0..2)
struct QueryCtx {
    V3 q;
    int kx, ky, kz;
};
__device__ __forceinline__ QueryCtx make_query(const V3 &q, double res, int lane) {
    const double c = lane == 0 ? q.x : (lane == 1 ? q.y : q.z);
    const int k = voxel_coord(c, res);
    QueryCtx ctx;
    ctx.q = q;
    ctx.kx = __shfl_sync(0xffffffffu, k, 0);
    ctx.ky = __shfl_sync(0xffffffffu, k, 1);
    ctx.kz = __shfl_sync(0xffffffffu, k, 2);
    return ctx;
}

// Returns the number of neighbors kept (<= kmax); lane l < n holds the l-th nearest in `best`.
// stage: 64 KnnStage entries of shared memory private to this warp.
//
// Memory-level parallelism: the stencil's points are addressed as ONE flattened list (prefix sum of the voxel
// counts over the lanes); chunk c gives lane l the candidate with flat index 32 c + l, found by a 5-step binary
// search over the prefix sums with shuffles. The loads of up to kPrefetch chunks are issued back to back before any
// of them is consumed, so a keypoint pays ~one L2/HBM round trip for all its map points instead of one per voxel.
// (Bench map, K = 1237: a stencil holds 147 points on average, median 153, p99 301 — with 4 chunks = 128 points per
// batch most keypoints need two batches; -DCTICP_PREFETCH=6 / 8 are experiment builds, tools/ab_variants.sh.)
#ifndef CTICP_PREFETCH
#define CTICP_PREFETCH 4
#endif
constexpr int kPrefetch = CTICP_PREFETCH;

// (Outlining this function — one copy of the sort / merge network instead of one per unrolled call site, a kernel about
// a sixth smaller — was measured slower.)
__device__ __forceinline__ void knn_consume32(KnnStage *stage, int &fill, KnnEntry &best, int lane) {
    const KnnStage t = stage[lane];
    KnnEntry c{t.d2, t.seq, t.addr};
    knn_sort32(c, lane);
    knn_merge32(best, c, lane);
    KnnStage rest = stage[32 + lane];   // garbage beyond fill-32 is never read back
    __syncwarp();
    stage[lane] = rest;
    fill -= 32;
    __syncwarp();
}

//
// kFilter: RadiusSearchInPlace with a sensor_location (map.h:482-490): a stored point whose (oriented) normal faces away
// from the sensor, (sensor - query) . normal < 0, is skipped. `to_sensor` = sensor_location - query.
template <bool kFilter = false>
__device__ __forceinline__ int warp_gather_knn(const GatherConfig &G, const int *stencil, const QueryCtx &ctx,
                                               int lane, KnnStage *stage, KnnEntry &best, unsigned &stencil_points,
                                               V3 to_sensor = V3{0, 0, 0}) {
    const MapLevel &L = G.L;
    const int side = 2 * G.r + 1;
    const int nst = side * side * side;
    const V3 &q = ctx.q;
    const int kx = ctx.kx, ky = ctx.ky, kz = ctx.kz;
    best.d2 = kKnnInf;
    best.seq = 0x7fffffff;
    best.addr = 0;
    int fill = 0;
    unsigned pts_total = 0;
    const unsigned lt_mask = (1u << lane) - 1u;
#ifdef CTICP_PRUNE
    // Opt-in (build with -DCTICP_PRUNE): distance of the kmax-th best so far — a later candidate at or beyond it can
    // never enter the result (candidates arrive in scan order, so on a tie the earlier-scanned point, already kept,
    // wins, map.h:495). Parity-clean (all GPU tests pass) but was neutral on config 2 (a
    // keypoint there has ~35 in-radius candidates, i.e. one or two merges either way); kept for denser maps.
    double prune_d2 = kKnnInf;
#endif

    for (int base = 0; base < nst; base += 32) {
        const int s = base + lane;
        int slot = 0;
        int cnt = 0;
        double ox = 0, oy = 0, oz = 0;   // my voxel's origin relative to the query (fp64)
        double sdn = 0;                  // kFilter: to_sensor . voxel normal
        int has_normal = 0;
        if (s < nst) {
            int dx, dy, dz;
            stencil_lookup(stencil, s, G.r, dx, dy, dz);
            uint32_t c = 0;
            const int found = map_find(L, pack_voxel(kx + dx, ky + dy, kz + dz), &c);
            if (found >= 0) {
                slot = found;
                cnt = (int) c;
                if (kFilter && L.normals && c > 0) {
                    const double *nrm = L.normals + 4 * (size_t) found;
                    if (nrm[3] != 0.0) {
                        has_normal = 1;
                        sdn = to_sensor.x * nrm[0] + to_sensor.y * nrm[1] + to_sensor.z * nrm[2];
                    }
                }
            }
            ox = (kx + dx) * L.res - q.x;
            oy = (ky + dy) * L.res - q.y;
            oz = (kz + dz) * L.res - q.z;
        }
        // inclusive prefix sum of the counts over the lanes
        int incl = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        const int total = __shfl_sync(0xffffffffu, incl, 31);
        const int excl = incl - cnt;
        pts_total += (unsigned) total;

        for (int c0 = 0; c0 < total; c0 += 32 * kPrefetch) {
            float4 pv[kPrefetch];
            int owner[kPrefetch];
            // phase 1: locate and issue every load of this batch
#pragma unroll
            for (int u = 0; u < kPrefetch; ++u) {
                const int f = c0 + 32 * u + lane;   // flat candidate index
                owner[u] = -1;
                pv[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (c0 + 32 * u < total) {           // warp-uniform
                    // owner = last lane whose exclusive prefix is <= f (binary search over lanes)
                    int lo = 0;
#pragma unroll
                    for (int step = 16; step > 0; step >>= 1) {
                        const int probe = lo + step;
                        const int ex = __shfl_sync(0xffffffffu, excl, probe & 31);
                        if (probe < 32 && ex <= f) lo = probe;
                    }
                    const int o_excl = __shfl_sync(0xffffffffu, excl, lo);
                    const int o_slot = __shfl_sync(0xffffffffu, slot, lo);
                    if (f < total) {
                        owner[u] = lo | ((f - o_excl) << 8);
                        pv[u] = __ldg(L.points + (size_t) o_slot * L.B + (f - o_excl));
                    }
                }
            }
            // phase 2: distances, radius test, compaction into the staging buffer, top-k maintenance
#pragma unroll
            for (int u = 0; u < kPrefetch; ++u) {
                if (c0 + 32 * u < total) {           // warp-uniform
                    const int ol = owner[u] < 0 ? 0 : (owner[u] & 0xff);
                    const double vx = __shfl_sync(0xffffffffu, ox, ol), vy = __shfl_sync(0xffffffffu, oy, ol),
                                 vz = __shfl_sync(0xffffffffu, oz, ol);
                    const int vslot = __shfl_sync(0xffffffffu, slot, ol);
                    const bool valid = owner[u] >= 0;
                    const int j = owner[u] >> 8;
                    const double rx = vx + f32_to_f64(pv[u].x), ry = vy + f32_to_f64(pv[u].y), rz = vz + f32_to_f64(pv[u].z);
                    const double d2 = rx * rx + ry * ry + rz * rz;
                    bool in = valid && !(d2 > G.radius2);
#ifdef CTICP_PRUNE
                    in = in && d2 < prune_d2;
#endif
                    if (kFilter) {
                        const double vs = __shfl_sync(0xffffffffu, sdn, ol);
                        const int vh = __shfl_sync(0xffffffffu, has_normal, ol);
                        // this point's copy of the normal is -n when its w is negative
                        const double scalar = signbit(pv[u].w) ? -vs : vs;
                        if (vh && scalar < 0.0) in = false;
                    }
                    const unsigned m = __ballot_sync(0xffffffffu, in);
                    if (in) {
                        KnnStage e;
                        e.d2 = d2;
                        e.seq = (base + ol) * 64 + j;   // scan order of the reference: stencil index, then index in voxel
                        e.addr = (uint32_t) ((size_t) vslot * L.B + j);
                        stage[fill + __popc(m & lt_mask)] = e;
                    }
                    fill += __popc(m);
                    __syncwarp();
                    if (fill >= 32) {
                        knn_consume32(stage, fill, best, lane);
#ifdef CTICP_PRUNE
                        prune_d2 = __shfl_sync(0xffffffffu, best.d2, G.kmax - 1);
#endif
                    }
                }
            }
        }
    }
    if (fill > 0) {
        KnnEntry c{kKnnInf, 0x7fffffff, 0};
        if (lane < fill) {
            const KnnStage t = stage[lane];
            c = KnnEntry{t.d2, t.seq, t.addr};
        }
        knn_sort32(c, lane);
        knn_merge32(best, c, lane);
    }
    __syncwarp();
    stencil_points = pts_total;
    const int found = __popc(__ballot_sync(0xffffffffu, best.d2 < kKnnInf));
    return found < G.kmax ? found : G.kmax;
}

// Neighbor position relative to the query, fp64, recomputed from the entry (stencil index in seq, offset at addr).
__device__ __forceinline__ V3 knn_rel_position(const GatherConfig &G, const int *stencil, const QueryCtx &ctx,
                                               const KnnEntry &e) {
    const MapLevel &L = G.L;
    int dx, dy, dz;
    stencil_lookup(stencil, e.seq >> 6, G.r, dx, dy, dz);
    const float4 p = __ldg(L.points + e.addr);
    return V3{((ctx.kx + dx) * L.res - ctx.q.x) + (double) p.x, ((ctx.ky + dy) * L.res - ctx.q.y) + (double) p.y,
              ((ctx.kz + dz) * L.res - ctx.q.z) + (double) p.z};
}

// ---- 3x3 symmetric eigen-decomposition (cyclic Jacobi, fp64, registers only) ---------------------------------
// Stand-in for Eigen::JacobiSVD<Matrix3d>(C, ComputeFullV) on a symmetric matrix (neighborhood.h:293): singular
// values = |eigenvalues| descending, normal = V.col(2).
#define CT_JACOBI_ROT(app, aqq, apq, arp, arq, v0p, v0q, v1p, v1q, v2p, v2q)          \
    if (apq != 0.0) {                                                                 \
        const double theta = (aqq - app) / (2.0 * apq);                               \
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0)); \
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;                          \
        app -= t * apq;                                                               \
        aqq += t * apq;                                                               \
        apq = 0.0;                                                                    \
        { const double x = arp, y = arq; arp = c * x - s * y; arq = s * x + c * y; }  \
        { const double x = v0p, y = v0q; v0p = c * x - s * y; v0q = s * x + c * y; }  \
        { const double x = v1p, y = v1q; v1p = c * x - s * y; v1q = s * x + c * y; }  \
        { const double x = v2p, y = v2q; v2p = c * x - s * y; v2q = s * x + c * y; }  \
    }

struct Eig3 {
    double sv0, sv1, sv2;   // |eigenvalues| descending
    V3 normal;              // eigenvector of sv2
};
struct Eig3Full {
    double sv0, sv1, sv2;
    V3 line, normal;        // eigenvectors of sv0 / sv2 (V.col(0), V.col(2))
};

static __device__ __noinline__ Eig3Full sym_eig3_full(double a00, double a01, double a02, double a11, double a12, double a22) {
    double v00 = 1, v01 = 0, v02 = 0, v10 = 0, v11 = 1, v12 = 0, v20 = 0, v21 = 0, v22 = 1;
#pragma unroll 1
    for (int sweep = 0; sweep < 12; ++sweep) {
        const double off = a01 * a01 + a02 * a02 + a12 * a12;
        const double diag = a00 * a00 + a11 * a11 + a22 * a22;
        if (off <= 1e-32 * diag || off == 0.0) break;
        CT_JACOBI_ROT(a00, a11, a01, a02, a12, v00, v01, v10, v11, v20, v21)   // (p,q)=(0,1), r=2
        CT_JACOBI_ROT(a00, a22, a02, a01, a12, v00, v02, v10, v12, v20, v22)   // (0,2), r=1
        CT_JACOBI_ROT(a11, a22, a12, a01, a02, v01, v02, v11, v12, v21, v22)   // (1,2), r=0
    }
    double e0 = fabs(a00), e1 = fabs(a11), e2 = fabs(a22);
    V3 c0{v00, v10, v20}, c1{v01, v11, v21}, c2{v02, v12, v22};
    // sort descending (stable like std::sort on 3 elements is irrelevant: values differ in practice)
    if (e0 < e1) { double t = e0; e0 = e1; e1 = t; V3 tv = c0; c0 = c1; c1 = tv; }
    if (e1 < e2) { double t = e1; e1 = e2; e2 = t; V3 tv = c1; c1 = c2; c2 = tv; }
    if (e0 < e1) { double t = e0; e0 = e1; e1 = t; V3 tv = c0; c0 = c1; c1 = tv; }
    return Eig3Full{e0, e1, e2, c0, c2};
}
__device__ __forceinline__ Eig3 sym_eig3(double a00, double a01, double a02, double a11, double a12, double a22) {
    const Eig3Full f = sym_eig3_full(a00, a01, a02, a11, a12, a22);
    return Eig3{f.sv0, f.sv1, f.sv2, f.normal};
}

// Non-iterative variant: eigenvalues from the trigonometric solution of the characteristic cubic, the eigenvector of
// the smallest one from the largest cross product of two rows of (A - e0 I) (D. Eberly, "A Robust Eigensolver for
// 3x3 Symmetric Matrices"). One acos + two cos instead of ~15 dependent Jacobi rotations: the dependent fp64 chain
// of the per-keypoint epilogue shrinks ~5x. The result is verified ((A - e0 I) n ~ 0); the rare failure (two
// coincident eigenvalues, where the normal is ill-defined anyway) falls back to the Jacobi solver.
// cos and sin on [0, pi/3] by their Taylor series (x^26 / x^25: truncation < 1e-26, measured error 1.1e-16 = libm's): the
// trigonometric eigenvalue formula needs cos(t) and cos(t + 2 pi / 3) = -cos(t)/2 - sin(t) sqrt(3)/2. libm's cos costs an
// argument reduction with two conversions on the XU pipe per call (se3.cuh).
__device__ __forceinline__ void cos_sin_upto_third_pi(double x, double &c, double &s) {
    const double x2 = x * x;
    double pc = -2.4795962632247976e-27, ps = 6.446950284384474e-26;
    pc = pc * x2 + 1.6117375710961184e-24;  ps = ps * x2 - 3.868170170630684e-23;
    pc = pc * x2 - 8.896791392450574e-22;   ps = ps * x2 + 1.9572941063391263e-20;
    pc = pc * x2 + 4.110317623312165e-19;   ps = ps * x2 - 8.22063524662433e-18;
    pc = pc * x2 - 1.5619206968586225e-16;  ps = ps * x2 + 2.8114572543455206e-15;
    pc = pc * x2 + 4.779477332387385e-14;   ps = ps * x2 - 7.647163731819816e-13;
    pc = pc * x2 - 1.1470745597729725e-11;  ps = ps * x2 + 1.6059043836821613e-10;
    pc = pc * x2 + 2.08767569878681e-09;    ps = ps * x2 - 2.505210838544172e-08;
    pc = pc * x2 - 2.755731922398589e-07;   ps = ps * x2 + 2.7557319223985893e-06;
    pc = pc * x2 + 2.48015873015873e-05;    ps = ps * x2 - 0.0001984126984126984;
    pc = pc * x2 - 0.001388888888888889;    ps = ps * x2 + 0.008333333333333333;
    pc = pc * x2 + 0.041666666666666664;    ps = ps * x2 - 0.16666666666666666;
    pc = pc * x2 - 0.5;                     ps = ps * x2 + 1.0;
    c = pc * x2 + 1.0;
    s = x * ps;
}

__device__ __forceinline__ Eig3 sym_eig3_fast(double a00, double a01, double a02, double a11, double a12, double a22) {
    const double mx = fmax(fmax(fmax(fabs(a00), fabs(a01)), fmax(fabs(a02), fabs(a11))), fmax(fabs(a12), fabs(a22)));
    if (!(mx > 0.0)) return sym_eig3(a00, a01, a02, a11, a12, a22);
    const double inv = 1.0 / mx;
    const double s00 = a00 * inv, s01 = a01 * inv, s02 = a02 * inv, s11 = a11 * inv, s12 = a12 * inv, s22 = a22 * inv;
    const double nrm = s01 * s01 + s02 * s02 + s12 * s12;
    if (!(nrm > 0.0)) return sym_eig3(a00, a01, a02, a11, a12, a22);
    const double q = (s00 + s11 + s22) * (1.0 / 3.0);
    const double b00 = s00 - q, b11 = s11 - q, b22 = s22 - q;
    const double p = sqrt((b00 * b00 + b11 * b11 + b22 * b22 + 2.0 * nrm) * (1.0 / 6.0));
    const double c00 = b11 * b22 - s12 * s12, c01 = s01 * b22 - s12 * s02, c02 = s01 * s12 - b11 * s02;
    const double det = (b00 * c00 - s01 * c01 + s02 * c02) / (p * p * p);
    const double half_det = fmin(fmax(det * 0.5, -1.0), 1.0);
    const double angle = acos(half_det) * (1.0 / 3.0);
    double ca, sa;   // angle in [0, pi/3]
    cos_sin_upto_third_pi(angle, ca, sa);
    const double beta2 = 2.0 * ca;
    const double beta0 = -ca - 1.7320508075688772 * sa;   // 2 cos(angle + 2 pi / 3)
    const double beta1 = -(beta0 + beta2);
    const double e0 = q + p * beta0, e1 = q + p * beta1, e2 = q + p * beta2;   // e0 <= e1 <= e2
    // rows of (A - e0 I)
    const V3 r0{s00 - e0, s01, s02}, r1{s01, s11 - e0, s12}, r2{s02, s12, s22 - e0};
    const V3 x01 = cross(r0, r1), x02 = cross(r0, r2), x12 = cross(r1, r2);
    const double d01 = dot(x01, x01), d02 = dot(x02, x02), d12 = dot(x12, x12);
    V3 n = x01;
    double dm = d01;
    if (d02 > dm) { n = x02; dm = d02; }
    if (d12 > dm) { n = x12; dm = d12; }
    if (!(dm > 0.0)) return sym_eig3(a00, a01, a02, a11, a12, a22);
    const double ninv = rsqrt(dm);
    n = ninv * n;
    // verification in scaled units (|A| ~ 1)
    const double rx = dot(r0, n), ry = dot(r1, n), rz = dot(r2, n);
    if (!(rx * rx + ry * ry + rz * rz < 1e-22)) return sym_eig3(a00, a01, a02, a11, a12, a22);
    double v0 = fabs(e2), v1 = fabs(e1), v2 = fabs(e0);
    // |eigenvalues| descending (a tiny negative e0 of a PSD matrix can only reorder within rounding noise)
    if (v0 < v1) { const double t = v0; v0 = v1; v1 = t; }
    if (v1 < v2) return sym_eig3(a00, a01, a02, a11, a12, a22);   // |e0| not the smallest: indefinite input, use Jacobi
    return Eig3{v0 * mx, v1 * mx, v2 * mx, n};
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

struct NeighborhoodDesc {
    V3 normal;       // unit normal (sign arbitrary)
    double a2D;
    V3 far_rel;      // farthest kept neighbor relative to the query (= reference points[0] - query)
    double far_d2;
};

// TNeighborhood::ComputeNeighborhood + ComputeNeighborhoodInfo on the n neighbors held one-per-lane.
// Covariance is accumulated CENTRED ON THE QUERY (the reference's uncentred E[xx^T]-mu mu^T in world coordinates,
// neighborhood.h:237-244, is the same quantity up to its own fp64 cancellation error).
__device__ __forceinline__ NeighborhoodDesc warp_describe(const GatherConfig &G, const int *stencil,
                                                          const QueryCtx &ctx, const KnnEntry &best, int n, int lane) {
    V3 rel{0, 0, 0};
    if (lane < n) rel = knn_rel_position(G, stencil, ctx, best);
    const double inv = 1.0 / (double) n;
    const double mx = warp_sum(rel.x) * inv, my = warp_sum(rel.y) * inv, mz = warp_sum(rel.z) * inv;
    const double cxx = warp_sum(rel.x * rel.x) * inv - mx * mx, cxy = warp_sum(rel.x * rel.y) * inv - mx * my,
                 cxz = warp_sum(rel.x * rel.z) * inv - mx * mz, cyy = warp_sum(rel.y * rel.y) * inv - my * my,
                 cyz = warp_sum(rel.y * rel.z) * inv - my * mz, czz = warp_sum(rel.z * rel.z) * inv - mz * mz;
    const Eig3 e = sym_eig3_fast(cxx, cxy, cxz, cyy, cyz, czz);
    NeighborhoodDesc d;
    d.normal = e.normal;
    d.a2D = (sqrt(e.sv1) - sqrt(e.sv2)) / sqrt(e.sv0);
    d.far_rel.x = __shfl_sync(0xffffffffu, rel.x, n - 1);
    d.far_rel.y = __shfl_sync(0xffffffffu, rel.y, n - 1);
    d.far_rel.z = __shfl_sync(0xffffffffu, rel.z, n - 1);
    d.far_d2 = __shfl_sync(0xffffffffu, best.d2, n - 1);
    return d;
}

// ComputeNeighborhood(ALL_BUT_KDTREE) for solver ROBUST (neighborhood.h:226-257, 286-316): everything above plus
// line = V.col(0), planarity, linearity, the covariance and the barycenter (relative to the query).
struct NeighborhoodDescFull {
    V3 normal, line, mean_rel, far_rel;
    double planarity, linearity;
    double cov[6];   // xx xy xz yy yz zz
};
__device__ __forceinline__ NeighborhoodDescFull warp_describe_full(const GatherConfig &G, const int *stencil,
                                                                   const QueryCtx &ctx, const KnnEntry &best, int n,
                                                                   int lane) {
    V3 rel{0, 0, 0};
    if (lane < n) rel = knn_rel_position(G, stencil, ctx, best);
    const double inv = 1.0 / (double) n;
    const double mx = warp_sum(rel.x) * inv, my = warp_sum(rel.y) * inv, mz = warp_sum(rel.z) * inv;
    NeighborhoodDescFull d;
    d.cov[0] = warp_sum(rel.x * rel.x) * inv - mx * mx;
    d.cov[1] = warp_sum(rel.x * rel.y) * inv - mx * my;
    d.cov[2] = warp_sum(rel.x * rel.z) * inv - mx * mz;
    d.cov[3] = warp_sum(rel.y * rel.y) * inv - my * my;
    d.cov[4] = warp_sum(rel.y * rel.z) * inv - my * mz;
    d.cov[5] = warp_sum(rel.z * rel.z) * inv - mz * mz;
    const Eig3Full e = sym_eig3_full(d.cov[0], d.cov[1], d.cov[2], d.cov[3], d.cov[4], d.cov[5]);
    d.normal = e.normal;
    d.line = e.line;
    d.linearity = (e.sv0 - e.sv1) / e.sv0;
    d.planarity = (e.sv1 - e.sv2) / e.sv0;
    d.mean_rel = V3{mx, my, mz};
    d.far_rel.x = __shfl_sync(0xffffffffu, rel.x, n - 1);
    d.far_rel.y = __shfl_sync(0xffffffffu, rel.y, n - 1);
    d.far_rel.z = __shfl_sync(0xffffffffu, rel.z, n - 1);
    return d;
}

}  // namespace cticp
