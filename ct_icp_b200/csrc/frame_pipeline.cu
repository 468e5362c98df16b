// frame_pipeline.cu — per-scan device pipeline around the ICP: ingest, voxel sub-sampling, keypoint grid sampling,
// continuous-time transform of the frame.
//
// Reference: Odometry::InitializeFrame (src/ct_icp/odometry.cpp:333-382), sub_sample_frame / grid_sampling
// (src/ct_icp/ct_icp.cpp:65-101), the post-registration transforms (odometry.cpp:463-486).
//
// Order contract (DESIGN.md): std::shuffle + "first point seen per voxel" becomes
//   winner(voxel) = argmin over the voxel's points of perm(i)        [64-bit atomicMin on (perm(i) << 32 | i)]
//   output order  = ascending perm(i) of the winners                   [flag array in permuted index space + scan]
// and the second shuffle is one scatter through a second permutation — no sort anywhere.
#include "frame_pipeline.h"

#include <cooperative_groups.h>
#include <cstdlib>

#include <algorithm>
#include <cstring>

namespace cticp {

#define CT_CUDA_CHECK(expr)                                                                              \
    do {                                                                                                 \
        cudaError_t _e = (expr);                                                                         \
        if (_e != cudaSuccess)                                                                           \
            throw CudaError(std::string(#expr) + ": " + cudaGetErrorString(_e) + " @" + __FILE__ + ":" + \
                            std::to_string(__LINE__));                                                   \
    } while (0)

constexpr unsigned long long kGridEmpty = ~0ull;
constexpr size_t kMaxTiles = 4096;   // up to 4M points per scan
constexpr int kTileShift = 10, kTile = 1 << kTileShift, kTileThreads = kTile / 4;   // 1024 positions per CTA
// d_desc_: the fused sampler's look-back descriptors (selection 1 | selection 2 | the capacity of grid 2 its last launch
// used), then the standalone selection's descriptors and tile ticket
constexpr size_t kFusedDescWords = 2 * kMaxTiles + 1, kDescWords = kFusedDescWords + kMaxTiles + 1;

// voxel key of sub_sample_frame: static_cast<short>(raw / size) per axis (ct_icp.cpp:70-72)
__device__ __forceinline__ unsigned long long short_voxel_key(const RawPoint &p, double voxel_size) {
    // int(p / size) from the reciprocal (division only next to an integer quotient: voxel_coord_rcp, device_map.cuh)
    const double inv = 1.0 / voxel_size;
    const short x = (short) voxel_coord_rcp(p.x, voxel_size, inv);
    const short y = (short) voxel_coord_rcp(p.y, voxel_size, inv);
    const short z = (short) voxel_coord_rcp(p.z, voxel_size, inv);
    return ((unsigned long long) (unsigned short) x << 32) | ((unsigned long long) (unsigned short) y << 16) |
           (unsigned long long) (unsigned short) z;
}

// find-or-insert the key in the hash grid, then bid `bid` (priority << 32 | index) for it; returns the slot
__device__ __forceinline__ uint32_t grid_bid(unsigned long long key, unsigned long long bid, unsigned long long *keys,
                                             unsigned long long *vals, uint32_t cap_mask) {
    uint32_t h = hash_key(key) & cap_mask;
    while (true) {
        unsigned long long k = *reinterpret_cast<volatile unsigned long long *>(&keys[h]);
        if (k == kGridEmpty) k = atomicCAS(&keys[h], kGridEmpty, key);
        if (k == kGridEmpty || k == key) break;
        h = (h + 1) & cap_mask;
    }
    atomicMin(&vals[h], bid);
    return h;
}
// claim: every point bids (priority, index) for its voxel and files its slot (and, permuted, its index) at its position
// p = priority, so that the selection can test the winners tile by tile in position order
__device__ __forceinline__ void grid_claim_dev(const float4 *pts, const float4 *lo, int n, double voxel_size, int use_perm,
                                               uint64_t seed, uint64_t counter, unsigned long long *keys,
                                               unsigned long long *vals, uint32_t cap_mask, int *__restrict__ slot_at,
                                               uint32_t *__restrict__ src) {
    const Perm perm = perm_make(seed, counter, (uint32_t) max(n, 1));
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned long long key = short_voxel_key(load_raw(pts, lo, i), voxel_size);
        const uint32_t prio = use_perm ? perm_apply(perm, (uint32_t) i) : (uint32_t) i;
        slot_at[prio] = (int) grid_bid(key, ((unsigned long long) prio << 32) | (unsigned) i, keys, vals, cap_mask);
        if (use_perm) src[prio] = (uint32_t) i;
    }
}
// n_host >= 0: the scan's N, known on the host only; this kernel leaves it in *n_store for the kernels behind it
__global__ void k_grid_claim(const float4 *__restrict__ pts, const float4 *__restrict__ lo, const int *__restrict__ d_n,
                             int n_host, int *n_store, double voxel_size, int use_perm, uint64_t seed, uint64_t counter,
                             unsigned long long *keys, unsigned long long *vals, uint32_t cap_mask, int *__restrict__ slot_at,
                             uint32_t *__restrict__ src) {
    if (n_host >= 0 && blockIdx.x == 0 && threadIdx.x == 0) *n_store = n_host;
    grid_claim_dev(pts, lo, n_host >= 0 ? n_host : *d_n, voxel_size, use_perm, seed, counter, keys, vals, cap_mask, slot_at, src);
}
// emit: compact the winners in permuted order and (optionally) scatter them through a second permutation (the
// second shuffle). One CTA per tile of 1024 positions: the exclusive prefix of a position is
//   Σ tile_count[tiles before] (every CTA re-adds those <= 512 counters) + a CTA-local scan of the tile's flags,
// which replaces a serial single-CTA scan over all positions by a fully parallel pass.
struct EmitScratch {
    uint32_t red[2][kTileThreads / 32];
    uint32_t warp[kTileThreads / 32];
    uint32_t before, total;
};
// all threads of a CTA of kTileThreads threads; returns the number of winners (identical in every CTA)
__device__ __forceinline__ uint32_t grid_emit_dev(const float4 *pts, const float4 *lo, const uint32_t *in_src_index, int n,
                                                  const uint32_t *flags, const uint32_t *src, const uint32_t *tile_count,
                                                  int use_perm2, uint64_t seed, uint64_t counter2, int override_alpha,
                                                  float alpha_value, float4 *__restrict__ out, float4 *__restrict__ out_lo,
                                                  uint32_t *__restrict__ out_src_index, int *__restrict__ d_total,
                                                  EmitScratch &sc) {
    uint32_t (&s_red)[2][kTileThreads / 32] = sc.red;
    uint32_t (&s_warp)[kTileThreads / 32] = sc.warp;
    uint32_t &s_before = sc.before, &s_total = sc.total;
    const int num_tiles = (n + kTile - 1) >> kTileShift;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    // grand total (domain of the second permutation) — identical in every CTA
    uint32_t tot = 0;
    for (int t = tid; t < num_tiles; t += kTileThreads) tot += tile_count[t];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
    if (lane == 0) s_red[1][w] = tot;
    __syncthreads();
    if (tid == 0) {
        uint32_t b = 0;
        for (int i = 0; i < kTileThreads / 32; ++i) b += s_red[1][i];
        s_total = b;
    }
    __syncthreads();
    const uint32_t total = s_total;
    if (blockIdx.x == 0 && tid == 0) *d_total = (int) total;
    const Perm perm2 = perm_make(seed, counter2, max(total, 1u));

    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        uint32_t before = 0;
        for (int t = tid; t < tile; t += kTileThreads) before += tile_count[t];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) before += __shfl_xor_sync(0xffffffffu, before, o);
        __syncthreads();   // s_red / s_warp reuse across tiles
        if (lane == 0) s_red[0][w] = before;
        // CTA-local exclusive scan of the tile's flags: 4 consecutive positions per thread
        const int p0 = (tile << kTileShift) + tid * 4;
        uint32_t v[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) v[k] = (p0 + k < n) ? flags[p0 + k] : 0u;
        const uint32_t tsum = v[0] + v[1] + v[2] + v[3];
        uint32_t incl = tsum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        if (lane == 31) s_warp[w] = incl;
        __syncthreads();
        if (tid == 0) {
            uint32_t b = 0;
            for (int i = 0; i < kTileThreads / 32; ++i) b += s_red[0][i];
            s_before = b;
            uint32_t run = 0;
            for (int i = 0; i < kTileThreads / 32; ++i) {
                const uint32_t c = s_warp[i];
                s_warp[i] = run;
                run += c;
            }
        }
        __syncthreads();
        uint32_t excl = s_before + s_warp[w] + (incl - tsum);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (v[k]) {
                const uint32_t dst = (use_perm2 && total > 1) ? perm_apply(perm2, excl) : excl;
                const uint32_t i = src[p0 + k];
                float4 val = pts[i];
                if (override_alpha) val.w = alpha_value;
                out[dst] = val;
                if (out_lo) {
                    float4 l = lo ? lo[i] : make_float4(0.f, 0.f, 0.f, 0.f);
                    if (override_alpha) l.w = 0.f;
                    out_lo[dst] = l;
                }
                out_src_index[dst] = in_src_index ? in_src_index[i] : i;
            }
            excl += v[k];
        }
    }
    return total;
}
__global__ void __launch_bounds__(kTileThreads)
k_grid_emit(const float4 *__restrict__ pts, const float4 *__restrict__ lo, const uint32_t *__restrict__ in_src_index,
            const int *__restrict__ d_n, const uint32_t *__restrict__ flags, const uint32_t *__restrict__ src,
            const uint32_t *__restrict__ tile_count, int use_perm2, uint64_t seed, uint64_t counter2,
            int override_alpha, float alpha_value, float4 *__restrict__ out, float4 *__restrict__ out_lo,
            uint32_t *__restrict__ out_src_index, int *__restrict__ d_total) {
    __shared__ EmitScratch sc;
    grid_emit_dev(pts, lo, in_src_index, *d_n, flags, src, tile_count, use_perm2, seed, counter2, override_alpha, alpha_value,
                  out, out_lo, out_src_index, d_total, sc);
}

// ---- single-pass selection: one CTA per tile of 1024 positions tests the winners of its positions (position p belongs to
// point i = src[p], or p itself without the first permutation; it won iff its bid is the minimum of its voxel), counts them,
// and gets the number of winners before the tile by decoupled look-back: the tile publishes its own count (status 1), walks
// back over the tiles before it adding their counts until it meets an inclusive prefix (status 2), and publishes its own
// inclusive prefix. desc[t] = status << 32 | value, one 64-bit word, so a reader never sees a status without its value.
// A tile only waits on tiles with smaller indices, which are processed by CTAs that are already running: the cooperative
// launch has every CTA resident and each CTA takes its tiles in ascending order; the standalone kernel hands tiles out
// in launch order from an atomic ticket.
__device__ __forceinline__ uint32_t tile_lookback(unsigned long long *desc, int tile, uint32_t count) {
    if (tile == 0) {
        atomicExch(&desc[0], (2ull << 32) | count);
        return 0u;
    }
    atomicExch(&desc[tile], (1ull << 32) | count);
    uint32_t before = 0;
    for (int t = tile - 1;;) {
        const unsigned long long d = *reinterpret_cast<volatile unsigned long long *>(&desc[t]);
        const uint32_t status = (uint32_t) (d >> 32);
        if (status == 0u) continue;
        before += (uint32_t) d;
        if (status == 2u) break;
        --t;
    }
    atomicExch(&desc[tile], (2ull << 32) | (before + count));
    return before;
}
// the winner at `i` goes to `dst` (alpha override: frames 0 and 1, odometry.cpp:355-359)
__device__ __forceinline__ void emit_point(const float4 *in, const float4 *in_lo, const uint32_t *in_src, uint32_t i, uint32_t dst,
                                           int override_alpha, float alpha_value, float4 *out, float4 *out_lo, uint32_t *out_src) {
    float4 val = in[i];
    if (override_alpha) val.w = alpha_value;
    out[dst] = val;
    if (out_lo) {
        float4 l = in_lo ? in_lo[i] : make_float4(0.f, 0.f, 0.f, 0.f);
        if (override_alpha) l.w = 0.f;
        out_lo[dst] = l;
    }
    out_src[dst] = in_src ? in_src[i] : i;
}
// one tile, all kTileThreads threads of the CTA. win != nullptr: the winners' point indices are compacted into win (a
// second permutation scatters them once their total is known); otherwise the winners themselves are written, compacted.
// The last tile writes the total to *d_total.
__device__ __forceinline__ void select_tile_dev(int tile, int n, const uint32_t *src, const int *slot_at,
                                                const unsigned long long *vals, unsigned long long *desc, int *d_total,
                                                uint32_t *win, const float4 *in, const float4 *in_lo, const uint32_t *in_src,
                                                float4 *out, float4 *out_lo, uint32_t *out_src, EmitScratch &sc) {
    uint32_t (&s_warp)[kTileThreads / 32] = sc.warp;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int p0 = (tile << kTileShift) + tid * 4;
    uint32_t idx[4], v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int p = p0 + k;
        idx[k] = 0u;
        v[k] = 0u;
        if (p < n) {
            idx[k] = src ? src[p] : (uint32_t) p;
            v[k] = vals[slot_at[p]] == (((unsigned long long) p << 32) | idx[k]) ? 1u : 0u;
        }
    }
    const uint32_t tsum = v[0] + v[1] + v[2] + v[3];
    uint32_t incl = tsum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    __syncthreads();   // s_warp / s_before reuse across tiles
    if (lane == 31) s_warp[w] = incl;
    __syncthreads();
    if (tid == 0) {
        uint32_t run = 0;
        for (int i = 0; i < kTileThreads / 32; ++i) {
            const uint32_t c = s_warp[i];
            s_warp[i] = run;
            run += c;
        }
        const uint32_t before = tile_lookback(desc, tile, run);
        sc.before = before;
        if (tile == ((n + kTile - 1) >> kTileShift) - 1) *d_total = (int) (before + run);
    }
    __syncthreads();
    uint32_t excl = sc.before + s_warp[w] + (incl - tsum);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (v[k]) {
            if (win) win[excl] = idx[k];
            else emit_point(in, in_lo, in_src, idx[k], excl, 0, 0.f, out, out_lo, out_src);
        }
        excl += v[k];
    }
}
// standalone selection (GridSelect): tiles from an atomic ticket (desc[kMaxTiles])
__global__ void __launch_bounds__(kTileThreads)
k_grid_select(const int *__restrict__ d_n, const uint32_t *__restrict__ src, const int *__restrict__ slot_at,
              const unsigned long long *__restrict__ vals, unsigned long long *desc, int *d_total, uint32_t *win,
              const float4 *__restrict__ in, const float4 *__restrict__ in_lo, const uint32_t *__restrict__ in_src,
              float4 *__restrict__ out, float4 *__restrict__ out_lo, uint32_t *__restrict__ out_src) {
    __shared__ EmitScratch sc;
    __shared__ int s_tile;
    const int n = *d_n, num_tiles = (n + kTile - 1) >> kTileShift;
    if (threadIdx.x == 0) s_tile = (int) atomicAdd(&desc[kMaxTiles], 1ull);
    __syncthreads();
    const int tile = s_tile;
    if (tile >= num_tiles) {
        if (tile == 0 && threadIdx.x == 0) *d_total = 0;
        return;
    }
    select_tile_dev(tile, n, src, slot_at, vals, desc, d_total, win, in, in_lo, in_src, out, out_lo, out_src, sc);
}
// the second shuffle: winner k (in first-permutation order) goes to perm2(k)
__global__ void k_grid_scatter(const int *__restrict__ d_total, const uint32_t *__restrict__ win, const float4 *__restrict__ in,
                               const float4 *__restrict__ in_lo, const uint32_t *__restrict__ in_src, uint64_t seed,
                               uint64_t counter2, int override_alpha, float alpha_value, float4 *__restrict__ out,
                               float4 *__restrict__ out_lo, uint32_t *__restrict__ out_src) {
    const uint32_t total = (uint32_t) *d_total;
    const Perm perm2 = perm_make(seed, counter2, max(total, 1u));
    for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < total; k += gridDim.x * blockDim.x)
        emit_point(in, in_lo, in_src, win[k], total > 1 ? perm_apply(perm2, k) : k, override_alpha, alpha_value, out, out_lo,
                   out_src);
}

// ---- both grid selections of a frame (sub_sample_frame N -> F, grid_sampling F -> K) in ONE cooperative launch, four
// phases and three grid barriers:
//   1. claim N points in grid 1 (priority = perm1(i)); clear the part of grid 2 the previous launch used
//   2. single-pass selection 1: the winners' indices, compacted in permuted order → win; F → counts[1]
//   3. winner k → frame[perm2(k)] (the second shuffle), and that frame point claims its voxel in grid 2 (priority = its
//      frame index)
//   4. single-pass selection 2 → keypoints; K → counts[2]. Grid 1 and the look-back descriptors of selection 1 are left
//      clean for the next launch (they are idle here), so a frame does not start with a 4 MB clear and a grid barrier.
struct FusedSampleArgs {
    const float4 *raw;
    const float4 *raw_lo;              // residual plane of the scan (nullptr: float32-representable)
    float4 *frame_lo, *kp_lo;          // residual planes of the two selections (written iff raw_lo)
    int n;                             // N (written to counts[0] for the kernels behind this one)
    int *counts;                       // [0] = N, [1] = F out, [2] = K out
    double voxel1, voxel2;
    uint64_t seed, c1, c2;
    int override_alpha;
    float alpha_value;
    unsigned long long *grid;          // selection 1: keys | vals, 2 * cap1 words
    uint32_t cap1;
    unsigned long long *grid2;         // selection 2: keys | vals, 2 * cap2 words (cap2 from F), clean between launches
    unsigned long long *desc;          // look-back descriptors: selection 1 | selection 2 | cap2 of the previous launch
    int *slot_at;                      // slot of each position (selection 1, then selection 2)
    uint32_t *src, *win;               // point of each position / compacted winners of selection 1
    float4 *frame, *keypoints;
    uint32_t *frame_src, *kp_src;
    // pre_cleared: the previous launch left grid 1 clean for at least this frame's capacity; clear_after: leave it clean
    int pre_cleared, clear_after;
};
__global__ void __launch_bounds__(kTileThreads, 4)
k_sample_fused(FusedSampleArgs a) {
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    __shared__ EmitScratch sc;
    const size_t gtid = (size_t) blockIdx.x * blockDim.x + threadIdx.x, gsize = (size_t) gridDim.x * blockDim.x;
    const int n = a.n, tiles1 = (n + kTile - 1) >> kTileShift;
    unsigned long long *desc1 = a.desc, *desc2 = a.desc + kMaxTiles, *cap2_used = a.desc + 2 * kMaxTiles;
    if (blockIdx.x == 0 && threadIdx.x == 0) a.counts[0] = n;
    if (!a.pre_cleared) {
        for (size_t i = gtid; i < 2 * (size_t) a.cap1; i += gsize) a.grid[i] = kGridEmpty;
        grid.sync();
    }
    // phase 1
    grid_claim_dev(a.raw, a.raw_lo, n, a.voxel1, 1, a.seed, a.c1, a.grid, a.grid + a.cap1, a.cap1 - 1, a.slot_at, a.src);
    const size_t prev2 = 2 * (size_t) *cap2_used;   // written in phase 3 of the previous launch
    for (size_t i = gtid; i < prev2; i += gsize) a.grid2[i] = kGridEmpty;
    for (size_t i = gtid; i < (size_t) tiles1; i += gsize) desc2[i] = 0ull;   // F <= N: selection 2 has at most tiles1 tiles
    grid.sync();
    // phase 2
    for (int tile = blockIdx.x; tile < tiles1; tile += gridDim.x)
        select_tile_dev(tile, n, a.src, a.slot_at, a.grid + a.cap1, desc1, a.counts + 1, a.win, nullptr, nullptr, nullptr,
                        nullptr, nullptr, nullptr, sc);
    if (tiles1 == 0 && blockIdx.x == 0 && threadIdx.x == 0) a.counts[1] = 0;
    grid.sync();
    // phase 3
    const uint32_t F = (uint32_t) *reinterpret_cast<volatile int *>(a.counts + 1);
    uint32_t cap2 = 1024;
    while (cap2 < 2 * F) cap2 <<= 1;
    if (blockIdx.x == 0 && threadIdx.x == 0) *cap2_used = cap2;
    float4 *frame_lo = a.raw_lo ? a.frame_lo : nullptr, *kp_lo = a.raw_lo ? a.kp_lo : nullptr;
    {
        const Perm perm2 = perm_make(a.seed, a.c2, max(F, 1u));
        for (uint32_t k = gtid; k < F; k += gsize) {
            const uint32_t i = a.win[k], j = F > 1 ? perm_apply(perm2, k) : k;
            emit_point(a.raw, a.raw_lo, nullptr, i, j, a.override_alpha, a.alpha_value, a.frame, frame_lo, a.frame_src);
            // the frame point's xyz is the raw point's (the override only touches alpha)
            const unsigned long long key = short_voxel_key(load_raw(a.raw, a.raw_lo, i), a.voxel2);
            a.slot_at[j] = (int) grid_bid(key, ((unsigned long long) j << 32) | j, a.grid2, a.grid2 + cap2, cap2 - 1);
        }
    }
    grid.sync();
    // phase 4
    const int tiles2 = (int) ((F + kTile - 1) >> kTileShift);
    for (int tile = blockIdx.x; tile < tiles2; tile += gridDim.x)
        select_tile_dev(tile, (int) F, nullptr, a.slot_at, a.grid2 + cap2, desc2, a.counts + 2, nullptr, a.frame, frame_lo,
                        a.frame_src, a.keypoints, kp_lo, a.kp_src, sc);
    if (tiles2 == 0 && blockIdx.x == 0 && threadIdx.x == 0) a.counts[2] = 0;
    for (size_t i = gtid; i < (size_t) tiles1; i += gsize) desc1[i] = 0ull;
    if (a.clear_after)
        for (size_t i = gtid; i < 2 * (size_t) a.cap1; i += gsize) a.grid[i] = kGridEmpty;
}
// ---- adaptive (distance-banded) grid sampling: AdaptiveSamplePointsInGrid, include/ct_icp/algorithm/sampling.h:55-110
struct AdaptiveBands {
    int num_bands;
    double distance[CTICP_MAX_ADAPTIVE_BANDS];
    double voxel_size[CTICP_MAX_ADAPTIVE_BANDS];
};
__device__ __forceinline__ int adaptive_band(const AdaptiveBands &B, const RawPoint &p, unsigned long long *key_out) {
    const double x = p.x, y = p.y, z = p.z;
    const double dist = sqrt(x * x + y * y + z * z);
    int lw = 0;   // std::lower_bound with comp(elem, v) = elem.first < v (:69-74)
    while (lw < B.num_bands && B.distance[lw] < dist) ++lw;
    if (!(dist >= B.distance[0] && dist < B.distance[B.num_bands - 1])) return -1;
    const int band = lw - 1;
    if (band < 0) return -1;
    const double vs = B.voxel_size[band];
    const int vx = voxel_coord(x, vs), vy = voxel_coord(y, vs), vz = voxel_coord(z, vs);   // slam::Voxel::Coordinates
    const int bias = 1 << 19;
    *key_out = ((unsigned long long) (band + 1) << 60) | ((unsigned long long) (unsigned) ((vx + bias) & 0xFFFFF) << 40) |
               ((unsigned long long) (unsigned) ((vy + bias) & 0xFFFFF) << 20) | (unsigned long long) (unsigned) ((vz + bias) & 0xFFFFF);
    return band;
}
__global__ void k_adaptive_claim(const float4 *__restrict__ pts, const float4 *__restrict__ lo, const int *__restrict__ d_n,
                                 int n_host, int *n_store, AdaptiveBands B, unsigned long long *keys,
                                 unsigned long long *vals, uint32_t cap_mask, int *__restrict__ slot_of,
                                 int *__restrict__ d_positions) {
    const int n = n_host >= 0 ? n_host : *d_n;   // (n_host: as k_grid_claim)
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        *d_positions = n * B.num_bands;
        if (n_host >= 0) *n_store = n_host;
    }
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        unsigned long long key;
        const int band = adaptive_band(B, load_raw(pts, lo, i), &key);
        if (band < 0) {
            slot_of[i] = -1;
            continue;
        }
        uint32_t h = hash_key(key) & cap_mask;
        while (true) {
            unsigned long long k = *reinterpret_cast<volatile unsigned long long *>(&keys[h]);
            if (k == kGridEmpty) k = atomicCAS(&keys[h], kGridEmpty, key);
            if (k == kGridEmpty || k == key) break;
            h = (h + 1) & cap_mask;
        }
        atomicMin(&vals[h], (unsigned long long) (unsigned) i);   // first seen = smallest index (:79-84)
        slot_of[i] = (int) h;
    }
}
__global__ void k_adaptive_mark(const float4 *__restrict__ pts, const float4 *__restrict__ lo, const int *__restrict__ d_n, AdaptiveBands B,
                                const unsigned long long *__restrict__ vals, const int *__restrict__ slot_of,
                                uint32_t *__restrict__ flags, uint32_t *__restrict__ src,
                                uint32_t *__restrict__ tile_count) {
    const int n = *d_n;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int slot = slot_of[i];
        if (slot < 0 || vals[slot] != (unsigned long long) (unsigned) i) continue;
        unsigned long long key;
        const int band = adaptive_band(B, load_raw(pts, lo, i), &key);
        const uint32_t pos = (uint32_t) band * (uint32_t) n + (uint32_t) i;   // band-major, then first appearance
        flags[pos] = 1u;
        src[pos] = (uint32_t) i;
        atomicAdd(&tile_count[pos >> kTileShift], 1u);
    }
}

// keypoints = frame (sampling NONE, odometry.cpp:546)
__global__ void k_copy_points(const float4 *__restrict__ in, const float4 *__restrict__ in_lo, const uint32_t *__restrict__ in_src,
                              const int *__restrict__ d_n, float4 *__restrict__ out, float4 *__restrict__ out_lo,
                              uint32_t *__restrict__ out_src, int *__restrict__ d_n_out) {
    const int n = *d_n;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        out[i] = in[i];
        if (in_lo) out_lo[i] = in_lo[i];
        out_src[i] = in_src[i];
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *d_n_out = n;
}
// max_num_keypoints: shuffle + resize (odometry.cpp:549-552) when *d_n > max_n
__global__ void k_truncate_shuffle(const float4 *__restrict__ in, const float4 *__restrict__ in_lo, const uint32_t *__restrict__ in_src,
                                   const int *__restrict__ d_n, int max_n, uint64_t seed, uint64_t counter,
                                   float4 *__restrict__ out, float4 *__restrict__ out_lo, uint32_t *__restrict__ out_src) {
    const int n = *d_n;
    const bool active = n > max_n;
    const Perm perm = perm_make(seed, counter, (uint32_t) max(n, 1));
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t d = active ? perm_apply(perm, (uint32_t) i) : (uint32_t) i;
        if (!active || (int) d < max_n) {
            out[d] = in[i];
            if (in_lo) out_lo[d] = in_lo[i];
            out_src[d] = in_src[i];
        }
    }
}
__global__ void k_clamp_count(int *d_n, int max_n) {
    if (*d_n > max_n) *d_n = max_n;
}
// world = ContinuousTransform(raw, begin, end, alpha) for every point (odometry.cpp:463-486)
// d_n == nullptr: n_host points
__global__ void k_transform_points(const float4 *__restrict__ pts, const float4 *__restrict__ lo, const int *__restrict__ d_n,
                                   int n_host, Q4 qb, V3 tb, Q4 qe, V3 te, SlerpConsts sc, double *__restrict__ world) {
    const int n = d_n ? *d_n : n_host;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const RawPoint p = load_raw(pts, lo, i);
        // acos / 1/sin(theta) of the pose pair are hoisted (sc): two sin per point instead of acos + three sin
        const V3 w = ct_transform_c(qb, tb, qe, te, p.alpha, V3{p.x, p.y, p.z}, sc);
        world[3 * i] = w.x; world[3 * i + 1] = w.y; world[3 * i + 2] = w.z;
    }
}

// DistortFrame (odometry.cpp:161-168): raw <- end^-1 * (Interpolate(begin, end, t) * raw), in place (alpha kept)
__global__ void k_distort_frame(float4 *__restrict__ pts, float4 *__restrict__ lo, int lo_valid,
                                const int *__restrict__ d_n, Q4 qb, V3 tb, Q4 qe, V3 te, SlerpConsts sc) {
    const int n = *d_n;
    const Q4 qi = qinverse(qe);
    const V3 ti = (-1.0) * qrot(qnormalized(qi), te);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const RawPoint p = load_raw(pts, lo_valid ? lo : nullptr, i);
        const V3 w = ct_transform_c(qb, tb, qe, te, p.alpha, V3{p.x, p.y, p.z}, sc);
        const V3 r = qrot(qnormalized(qi), w) + ti;
        store_raw(pts, lo, i, r.x, r.y, r.z, p.alpha);   // the distorted point is not float32-representable: hi + lo
    }
}

// ---------------------------------------------------------------------------------------------------------------
static uint32_t NextPow2(uint64_t v) {
    uint64_t p = 1;
    while (p < v) p <<= 1;
    return (uint32_t) p;
}

FramePipeline::FramePipeline(size_t max_points, cudaStream_t stream) : stream_(stream), max_points_(max_points) {
    const size_t n = max_points_;
    if (const char *e = getenv("CTICP_SAMPLE_PRECLEAR")) preclear_ = atoi(e) != 0;
    grid_cap_ = std::max<uint32_t>(NextPow2(2 * n), 1024);
    CT_CUDA_CHECK(cudaMallocHost(&h_stage_, sizeof(float4) * n));
    CT_CUDA_CHECK(cudaMallocHost(&h_counts_, sizeof(int) * 8));
    CT_CUDA_CHECK(cudaMalloc(&d_raw_, sizeof(float4) * n));
    raw_ptr_ = d_raw_;
    CT_CUDA_CHECK(cudaMalloc(&d_frame_, sizeof(float4) * n));
    CT_CUDA_CHECK(cudaMalloc(&d_keypoints_, sizeof(float4) * n));
    CT_CUDA_CHECK(cudaMalloc(&d_tmp_points_, sizeof(float4) * n));
    CT_CUDA_CHECK(cudaMalloc(&d_frame_src_, sizeof(uint32_t) * n));
    CT_CUDA_CHECK(cudaMalloc(&d_kp_src_, sizeof(uint32_t) * n));
    CT_CUDA_CHECK(cudaMalloc(&d_tmp_src_, sizeof(uint32_t) * n));
    CT_CUDA_CHECK(cudaMalloc(&d_grid_, sizeof(unsigned long long) * 2 * (size_t) grid_cap_));
    CT_CUDA_CHECK(cudaMalloc(&d_slot_of_, sizeof(int) * n));
    if ((n + kTile - 1) / kTile > kMaxTiles) throw std::invalid_argument("max_points_per_frame too large");
    CT_CUDA_CHECK(cudaMalloc(&d_win_, sizeof(uint32_t) * n));
    CT_CUDA_CHECK(cudaMalloc(&d_desc_, sizeof(unsigned long long) * kDescWords));
    CT_CUDA_CHECK(cudaMemsetAsync(d_desc_, 0, sizeof(unsigned long long) * kDescWords, stream_));
    CT_CUDA_CHECK(cudaMalloc(&d_src_, sizeof(uint32_t) * n));
    CT_CUDA_CHECK(cudaMalloc(&d_counts_, sizeof(int) * 8));
    CT_CUDA_CHECK(cudaMalloc(&d_frame_world_, sizeof(double) * 3 * n));
    CT_CUDA_CHECK(cudaMemsetAsync(d_counts_, 0, sizeof(int) * 8, stream_));
    memset(h_counts_, 0, sizeof(int) * 8);
}
FramePipeline::~FramePipeline() {
    cudaFreeHost(h_stage_); cudaFreeHost(h_counts_);
    cudaFree(d_raw_); cudaFree(d_frame_); cudaFree(d_keypoints_); cudaFree(d_tmp_points_);
    cudaFreeHost(h_stage_lo_);
    cudaFree(d_raw_lo_); cudaFree(d_frame_lo_); cudaFree(d_kp_lo_); cudaFree(d_tmp_lo_);
    cudaFree(d_frame_src_); cudaFree(d_kp_src_); cudaFree(d_tmp_src_);
    cudaFree(d_grid_); cudaFree(d_slot_of_); cudaFree(d_win_); cudaFree(d_desc_); cudaFree(d_src_);
    cudaFree(d_counts_); cudaFree(d_frame_world_); cudaFree(d_all_world_); cudaFree(d_adaptive_);
    cudaFree(d_grid2_);
}

int FramePipeline::Blocks(size_t n) const { return (int) std::max<size_t>(1, std::min<size_t>((n + 255) / 256, 132 * 8)); }

void FramePipeline::EnsureLo() {
    if (d_raw_lo_) return;
    CT_CUDA_CHECK(cudaMallocHost(&h_stage_lo_, sizeof(float4) * max_points_));
    CT_CUDA_CHECK(cudaMalloc(&d_raw_lo_, sizeof(float4) * max_points_));
    CT_CUDA_CHECK(cudaMalloc(&d_frame_lo_, sizeof(float4) * max_points_));
    CT_CUDA_CHECK(cudaMalloc(&d_kp_lo_, sizeof(float4) * max_points_));
    CT_CUDA_CHECK(cudaMalloc(&d_tmp_lo_, sizeof(float4) * max_points_));
}

void FramePipeline::UploadLo(size_t n) {
    EnsureLo();
    CT_CUDA_CHECK(cudaMemcpyAsync(d_raw_lo_, h_stage_lo_, sizeof(float4) * n, cudaMemcpyHostToDevice, stream_));
    raw_lo_ = true;
    raw_lo_ptr_ = d_raw_lo_;
    h2d_bytes_ += sizeof(float4) * n;
}

void FramePipeline::BeginScan(size_t n) {
    if (n > max_points_) throw CapacityError("scan has more points than max_points_per_frame");
    raw_lo_ = frame_lo_ = distorted_ = false;
    n_ = n;
    h_counts_[0] = (int) n;
    n_on_device_ = false;
    raw_ptr_ = d_raw_;
    raw_lo_ptr_ = d_raw_lo_;
}

int FramePipeline::TakeHostN(const int *d_n) {
    if (d_n != d_counts_ || n_on_device_) return -1;
    n_on_device_ = true;
    return (int) n_;
}

void FramePipeline::Upload(size_t n) {
    BeginScan(n);
    CT_CUDA_CHECK(cudaMemcpyAsync(d_raw_, h_stage_, sizeof(float4) * n, cudaMemcpyHostToDevice, stream_));
    h2d_bytes_ = sizeof(float4) * n;
}

void FramePipeline::UploadBegin(size_t n) {
    BeginScan(n);
    h2d_bytes_ = sizeof(float4) * n;
}
void FramePipeline::UploadRange(size_t begin, size_t end) {
    if (end <= begin) return;
    CT_CUDA_CHECK(cudaMemcpyAsync(d_raw_ + begin, h_stage_ + begin, sizeof(float4) * (end - begin), cudaMemcpyHostToDevice, stream_));
}

void FramePipeline::UploadFromDevice(const float4 *d_src, const float4 *d_src_lo, size_t n) {
    BeginScan(n);
    raw_ptr_ = d_src;
    raw_lo_ptr_ = d_src_lo;
    raw_lo_ = d_src_lo != nullptr;
    h2d_bytes_ = 0;
}

void FramePipeline::DetachRaw() {
    if (raw_ptr_ == d_raw_) return;
    if (n_) CT_CUDA_CHECK(cudaMemcpyAsync(d_raw_, raw_ptr_, sizeof(float4) * n_, cudaMemcpyDeviceToDevice, stream_));
    if (raw_lo_) {
        EnsureLo();
        CT_CUDA_CHECK(cudaMemcpyAsync(d_raw_lo_, raw_lo_ptr_, sizeof(float4) * n_, cudaMemcpyDeviceToDevice, stream_));
    }
    raw_ptr_ = d_raw_;
    raw_lo_ptr_ = d_raw_lo_;
}

void FramePipeline::GridSelect(const float4 *in, const float4 *in_lo, const uint32_t *in_src, const int *d_n_in,
                               size_t n_upper, double voxel_size, int use_perm1, uint64_t seed, uint64_t c1,
                               int use_perm2, uint64_t c2, int override_alpha, float alpha_value, float4 *out,
                               float4 *out_lo, uint32_t *out_src, int *d_n_out) {
    if (!in_lo) out_lo = nullptr;
    clean_cap_ = 0;   // (this selection dirties what the fused sampler may have left clean)
    // scratch hash grid: only the prefix that can be touched is cleared; keys and vals are adjacent → one memset
    const uint32_t cap = std::max<uint32_t>(NextPow2(2 * n_upper), 1024);
    unsigned long long *keys = d_grid_, *vals = d_grid_ + cap;
    CT_CUDA_CHECK(cudaMemsetAsync(keys, 0xFF, sizeof(unsigned long long) * 2 * (size_t) cap, stream_));
    // look-back descriptors + ticket of the standalone selection (the fused sampler's are kept apart: it relies on finding
    // its own clean)
    const size_t num_tiles = (n_upper + kTile - 1) / kTile;
    unsigned long long *desc = d_desc_ + kFusedDescWords;
    CT_CUDA_CHECK(cudaMemsetAsync(desc, 0, sizeof(unsigned long long) * (kMaxTiles + 1), stream_));
    const int n_host = TakeHostN(d_n_in);
    k_grid_claim<<<Blocks(n_upper), 256, 0, stream_>>>(in, in_lo, d_n_in, n_host, d_counts_, voxel_size, use_perm1, seed, c1,
                                                       keys, vals, cap - 1, d_slot_of_, d_src_);
    k_grid_select<<<(int) std::max<size_t>(1, num_tiles), kTileThreads, 0, stream_>>>(
        d_n_in, use_perm1 ? d_src_ : nullptr, d_slot_of_, vals, desc, d_n_out, use_perm2 ? d_win_ : nullptr, in, in_lo, in_src,
        out, out_lo, out_src);
    launches_ += 2;
    if (use_perm2) {
        k_grid_scatter<<<Blocks(n_upper), 256, 0, stream_>>>(d_n_out, d_win_, in, in_lo, in_src, seed, c2, override_alpha,
                                                             alpha_value, out, out_lo, out_src);
        launches_ += 1;
    }
    CT_CUDA_CHECK(cudaGetLastError());
}

void FramePipeline::AdaptiveSelect(const cticp_adaptive_options &o, const float4 *in, const float4 *in_lo,
                                   const uint32_t *in_src, const int *d_n_in, size_t n_upper, float4 *out,
                                   float4 *out_lo, uint32_t *out_src, int *d_n_out) {
    if (!in_lo) out_lo = nullptr;
    clean_cap_ = 0;
    if (o.num_points_per_voxel != 1) throw std::invalid_argument("adaptive sampling: only num_points_per_voxel == 1 is built");
    if (o.num_bands < 2 || o.num_bands > CTICP_MAX_ADAPTIVE_BANDS) throw std::invalid_argument("adaptive sampling: num_bands");
    AdaptiveBands B;
    B.num_bands = o.num_bands;
    for (int i = 0; i < CTICP_MAX_ADAPTIVE_BANDS; ++i) {
        B.distance[i] = o.distance[i];
        B.voxel_size[i] = o.voxel_size[i];
    }
    const size_t positions = n_upper * (size_t) o.num_bands;
    if ((positions + kTile - 1) / kTile > kMaxTiles) throw CapacityError("adaptive sampling: scan too large");
    if (positions > adaptive_capacity_) {
        CT_CUDA_CHECK(cudaStreamSynchronize(stream_));
        cudaFree(d_adaptive_);
        CT_CUDA_CHECK(cudaMalloc(&d_adaptive_, sizeof(uint32_t) * (kMaxTiles + 2 * positions)));
        adaptive_capacity_ = positions;
    }
    uint32_t *tile_count = d_adaptive_, *flags = d_adaptive_ + kMaxTiles, *src = flags + positions;
    const uint32_t cap = std::max<uint32_t>(NextPow2(2 * n_upper), 1024);
    unsigned long long *keys = d_grid_, *vals = d_grid_ + cap;
    CT_CUDA_CHECK(cudaMemsetAsync(keys, 0xFF, sizeof(unsigned long long) * 2 * (size_t) cap, stream_));
    CT_CUDA_CHECK(cudaMemsetAsync(tile_count, 0, sizeof(uint32_t) * (kMaxTiles + positions), stream_));
    const int blocks = Blocks(n_upper);
    int *d_positions = d_counts_ + 3;
    k_adaptive_claim<<<blocks, 256, 0, stream_>>>(in, in_lo, d_n_in, TakeHostN(d_n_in), d_counts_, B, keys, vals, cap - 1,
                                                  d_slot_of_, d_positions);
    k_adaptive_mark<<<blocks, 256, 0, stream_>>>(in, in_lo, d_n_in, B, vals, d_slot_of_, flags, src, tile_count);
    const size_t num_tiles = (positions + kTile - 1) / kTile;
    k_grid_emit<<<(int) std::min<size_t>(std::max<size_t>(1, num_tiles), 1184), kTileThreads, 0, stream_>>>(
        in, in_lo, in_src, d_positions, flags, src, tile_count, 0, 0, 0, 0, 0.f, out, out_lo, out_src, d_n_out);
    launches_ += 3;
    if (o.max_num_points > 0) {   // `indices.size() > kMaxNumPoints` lets max + 1 through (:96-105)
        k_clamp_count<<<1, 1, 0, stream_>>>(d_n_out, o.max_num_points + 1);
        launches_ += 1;
    }
    CT_CUDA_CHECK(cudaGetLastError());
}

// SubSampleFrame + SampleKeypoints(GRID) of one frame in a single cooperative launch (k_sample_fused). The keypoint
// sampling's parameters must be known when the frame arrives: true for the first registration attempt of a frame.
void FramePipeline::SampleFused(double voxel_size, double sample_voxel_size, uint64_t seed, uint64_t counter1,
                                uint64_t counter2, bool override_alpha, float alpha_value) {
    if (!d_grid2_) {
        CT_CUDA_CHECK(cudaMalloc(&d_grid2_, sizeof(unsigned long long) * 2 * (size_t) grid_cap_));
        CT_CUDA_CHECK(cudaMemsetAsync(d_grid2_, 0xFF, sizeof(unsigned long long) * 2 * (size_t) grid_cap_, stream_));
        int per_sm = 0;
        CT_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_sample_fused, kTileThreads, 0));
        int dev = 0, sms = 132;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        int want = 4;   // CTAs per SM: more hide the latency of the probes, fewer make the grid barriers cheaper (A/B knob)
        if (const char *e = getenv("CTICP_SAMPLE_CTAS_PER_SM")) want = std::max(1, atoi(e));
        fused_grid_ = std::max(1, std::min(per_sm, want) * sms);
    }
    FusedSampleArgs a;
    a.raw = raw_ptr_;
    a.raw_lo = d_raw_lo();
    a.n = (int) n_;
    n_on_device_ = true;
    a.frame_lo = d_frame_lo_; a.kp_lo = d_kp_lo_;
    frame_lo_ = raw_lo_;
    a.counts = d_counts_;
    a.voxel1 = voxel_size;
    a.voxel2 = sample_voxel_size;
    a.seed = seed; a.c1 = counter1; a.c2 = counter2;
    a.override_alpha = override_alpha ? 1 : 0;
    a.alpha_value = alpha_value;
    a.grid = d_grid_;
    a.cap1 = std::max<uint32_t>(NextPow2(2 * n_), 1024);
    a.pre_cleared = (preclear_ && clean_cap_ >= a.cap1) ? 1 : 0;
    a.clear_after = preclear_ ? 1 : 0;
    clean_cap_ = preclear_ ? a.cap1 : 0;        // what this launch leaves behind
    a.grid2 = d_grid2_;
    a.desc = d_desc_;
    a.slot_at = d_slot_of_;
    a.src = d_src_; a.win = d_win_;
    a.frame = d_frame_; a.keypoints = d_keypoints_;
    a.frame_src = d_frame_src_; a.kp_src = d_kp_src_;
    void *args[] = {&a};
    CT_CUDA_CHECK(cudaLaunchCooperativeKernel((void *) k_sample_fused, dim3(fused_grid_), dim3(kTileThreads), args, 0, stream_));
    launches_ += 1;
}

void FramePipeline::SubSampleFrame(double voxel_size, uint64_t seed, uint64_t counter1, uint64_t counter2,
                                   bool override_alpha, float alpha_value) {
    GridSelect(raw_ptr_, d_raw_lo(), nullptr, d_counts_ + 0, n_, voxel_size, 1, seed, counter1, 1, counter2,
               override_alpha ? 1 : 0, alpha_value, d_frame_, d_frame_lo_, d_frame_src_, d_counts_ + 1);
    frame_lo_ = raw_lo_;
}

void FramePipeline::SampleKeypoints(int sampling, double sample_voxel_size, int max_num_keypoints, uint64_t seed,
                                    uint64_t counter, const cticp_adaptive_options *adaptive) {
    if (sampling == CTICP_SAMPLING_ADAPTIVE) {
        if (!adaptive) throw std::invalid_argument("adaptive options missing");
        AdaptiveSelect(*adaptive, d_frame_, d_frame_lo(), d_frame_src_, d_counts_ + 1, n_, d_keypoints_, d_kp_lo_, d_kp_src_,
                       d_counts_ + 2);
    } else if (sampling == CTICP_SAMPLING_GRID) {
        GridSelect(d_frame_, d_frame_lo(), d_frame_src_, d_counts_ + 1, n_, sample_voxel_size, 0, 0, 0, 0, 0, 0, 0.f,
                   d_keypoints_, d_kp_lo_, d_kp_src_, d_counts_ + 2);
    } else {
        k_copy_points<<<Blocks(n_), 256, 0, stream_>>>(d_frame_, d_frame_lo(), d_frame_src_, d_counts_ + 1, d_keypoints_,
                                                       d_kp_lo_, d_kp_src_, d_counts_ + 2);
        launches_ += 1;
    }
    if (max_num_keypoints > 0) {
        k_truncate_shuffle<<<Blocks(n_), 256, 0, stream_>>>(d_keypoints_, d_keypoints_lo(), d_kp_src_, d_counts_ + 2,
                                                            max_num_keypoints, seed, counter, d_tmp_points_, d_tmp_lo_,
                                                            d_tmp_src_);
        k_clamp_count<<<1, 1, 0, stream_>>>(d_counts_ + 2, max_num_keypoints);
        std::swap(d_keypoints_, d_tmp_points_);
        std::swap(d_kp_lo_, d_tmp_lo_);
        std::swap(d_kp_src_, d_tmp_src_);
        launches_ += 2;
    }
    CT_CUDA_CHECK(cudaGetLastError());
}

void FramePipeline::QueueCountsReadback() {
    CT_CUDA_CHECK(cudaMemcpyAsync(h_counts_, d_counts_, sizeof(int) * 4, cudaMemcpyDeviceToHost, stream_));
}

void FramePipeline::DistortFrame(const Q4 &qb, const V3 &tb, const Q4 &qe, const V3 &te) {
    EnsureLo();
    k_distort_frame<<<Blocks(n_), 256, 0, stream_>>>(d_frame_, d_frame_lo_, frame_lo_ ? 1 : 0, d_counts_ + 1, qb, tb, qe, te,
                                                     slerp_consts(qb, qe));
    frame_lo_ = distorted_ = true;
    launches_ += 1;
    CT_CUDA_CHECK(cudaGetLastError());
}

void FramePipeline::TransformFrame(const Q4 &qb, const V3 &tb, const Q4 &qe, const V3 &te) {
    k_transform_points<<<Blocks(n_), 256, 0, stream_>>>(d_frame_, d_frame_lo(), d_counts_ + 1, 0, qb, tb, qe, te, slerp_consts(qb, qe), d_frame_world_);
    launches_ += 1;
    CT_CUDA_CHECK(cudaGetLastError());
}

void FramePipeline::EnsureAllWorld() {
    if (!d_all_world_) CT_CUDA_CHECK(cudaMalloc(&d_all_world_, sizeof(double) * 3 * max_points_));
}
void FramePipeline::TransformAll(const Q4 &qb, const V3 &tb, const Q4 &qe, const V3 &te, cudaStream_t stream) {
    EnsureAllWorld();
    k_transform_points<<<Blocks(n_), 256, 0, stream ? stream : stream_>>>(raw_ptr_, d_raw_lo(), nullptr, (int) n_, qb, tb, qe, te, slerp_consts(qb, qe), d_all_world_);
    launches_ += 1;
    CT_CUDA_CHECK(cudaGetLastError());
}

void FramePipeline::TransformInto(const float4 *pts, const float4 *lo, const int *d_n, const Q4 &qb, const V3 &tb,
                                  const Q4 &qe, const V3 &te, double *d_world, cudaStream_t stream) {
    k_transform_points<<<Blocks(n_), 256, 0, stream ? stream : stream_>>>(pts, lo, d_n, 0, qb, tb, qe, te, slerp_consts(qb, qe), d_world);
    launches_ += 1;
    CT_CUDA_CHECK(cudaGetLastError());
}

}  // namespace cticp
