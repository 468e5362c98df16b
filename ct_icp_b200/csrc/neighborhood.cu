// neighborhood.cu — slam::TNeighborhood (include/SlamCore/experimental/neighborhood.h): k-nearest search and neighbourhood
// description over any point set.
//
// Build (one pass of the world-cloud kind): load the points in fp64 and their bounding box (non-finite ones rejected),
// choose the cell size (below), key every point by its cell, claim the cell in an open-addressed table and count it,
// give each cell a range of the cell-ordered array, scatter the points into their ranges, then put each cell's points
// back into input order. Where a cell's range lies follows the schedule (an atomic counter hands the ranges out); no
// result depends on it, because the search ranks by (d2, index) and visits whole cells.
//
// Cell size: h0 = cbrt(V 8 / n) for the n valid points in a box of volume V (each side at least 2^-10 of the longest, so
// flat and straight clouds keep a finite count of cells): 8 points per cell on average if the points filled the box.
// When the occupied cells of h0 hold more than 16 points on average (points on surfaces, as in lidar maps), the size
// shrinks once to h0 sqrt(8 / mean): the factor that brings a surface back to 8 points per cell. Every cell size is at
// least the longest side / (2^21 - 2), so a cell coordinate fits 21 bits.
//
// Search: one warp per query; the k nearest so far are held one per lane, sorted by (d2, index) (gather.cuh's
// knn_sort32 / knn_merge32). The warp visits the cells at Chebyshev distance r = r0, r0 + 1, ... from the query's cell,
// where r0 is the first ring that meets the grid's box (the box is the coarse occupancy level: a query 10 km off the
// cloud starts at the cloud, not at its own cell). Before ring r it stops when k are held and the ring's lower bound on
// d2 exceeds the k-th d2 strictly (a later point at the same d2 with a lower index is never missed), or when the bound
// reaches max_radius. Describe runs the same search, then sums its neighbours' offsets from the query in list order.
#include "neighborhood.h"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <stdexcept>
#include <string>
#include <vector>

#include "device_checks.h"
#include "device_map.cuh"
#include "device_map.h"
#include "engine.h"
#include "gather.cuh"
#include "record_io.cuh"
#include "world_cloud.h"

namespace cticp {

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr double kCellTarget = 8.0;
constexpr int kMaxCell = (1 << 21) - 2;      // cells per axis - 1
constexpr int kListCap = 64;                 // a warp's staged cells
constexpr uint32_t kNoSlot = 0xFFFFFFFFu;

// the device variants read and write whole scalars: a misaligned pointer is refused, not left to fault in the kernel
void RequireAligned(const void *p, uint64_t align, const char *what) {
    if (reinterpret_cast<uintptr_t>(p) % align)
        throw std::invalid_argument(std::string(what) + ": not aligned to " + std::to_string(align) + " bytes");
}

int Blocks(uint64_t n) { return (int) std::max<uint64_t>(1, std::min<uint64_t>((n + kThreads - 1) / kThreads, 132 * 16)); }
int WarpBlocks(uint64_t m) { return (int) std::max<uint64_t>(1, std::min<uint64_t>((m + kWarps - 1) / kWarps, 132 * 64)); }

uint64_t Pow2AtLeast(uint64_t n) {
    uint64_t p = 1;
    while (p < n) p <<= 1;
    return p;
}

__device__ __forceinline__ bool finite3(double x, double y, double z) {
    return isfinite(x) && isfinite(y) && isfinite(z);
}

// the squared distance in the reference's order of operations, without FMA contraction: ((dx dx + dy dy) + dz dz)
__host__ __device__ __forceinline__ double dist2(double qx, double qy, double qz, double px, double py, double pz) {
#ifdef __CUDA_ARCH__
    const double dx = __dsub_rn(qx, px), dy = __dsub_rn(qy, py), dz = __dsub_rn(qz, pz);
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
#else
    const double dx = qx - px, dy = qy - py, dz = qz - pz;
    return (dx * dx + dy * dy) + dz * dz;
#endif
}

struct GridArgs {
    const ulonglong2 *table;
    uint64_t mask;
    const double4 *cpts;
    double ox, oy, oz, h, inv;
    int nx, ny, nz;
    int empty;   // no valid point
};

__device__ __forceinline__ unsigned long long cell_key(long long x, long long y, long long z) {
    return ((unsigned long long) x << 42) | ((unsigned long long) y << 21) | (unsigned long long) z;
}
__device__ __forceinline__ int cell_of(double p, double o, double inv, int dim) {
    const double c = floor((p - o) * inv);
    return c <= 0.0 ? 0 : c >= (double) (dim - 1) ? dim - 1 : (int) c;
}

// step 1: points (x, y, z of XT) to fp64 in index order; per-block bounding box of the finite ones and their count
template <typename XT, int LOAD>
__global__ void __launch_bounds__(kThreads) k_load(const unsigned char *xyz, uint64_t stride, uint64_t n,
                                                   double4 *__restrict__ ipts, double *__restrict__ bbox,
                                                   unsigned long long *__restrict__ rejected) {
    __shared__ double s_b[6][kThreads];
    __shared__ unsigned s_rej;
    if (threadIdx.x == 0) s_rej = 0;
    __syncthreads();
    double b[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};
    unsigned rej = 0;
    for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < n; i += (uint64_t) gridDim.x * blockDim.x) {
        XT x, y, z;
        load_xyz<XT, LOAD>(xyz + i * stride, x, y, z);
        const double px = (double) x, py = (double) y, pz = (double) z;
        ipts[i] = make_double4(px, py, pz, 0.0);
        if (!finite3(px, py, pz)) {
            ++rej;
            continue;
        }
        b[0] = fmin(b[0], px); b[1] = fmin(b[1], py); b[2] = fmin(b[2], pz);
        b[3] = fmax(b[3], px); b[4] = fmax(b[4], py); b[5] = fmax(b[5], pz);
    }
    if (rej) atomicAdd(&s_rej, rej);
#pragma unroll
    for (int a = 0; a < 6; ++a) s_b[a][threadIdx.x] = b[a];
    __syncthreads();
    for (int w = kThreads / 2; w > 0; w >>= 1) {
        if ((int) threadIdx.x < w) {
#pragma unroll
            for (int a = 0; a < 3; ++a) s_b[a][threadIdx.x] = fmin(s_b[a][threadIdx.x], s_b[a][threadIdx.x + w]);
#pragma unroll
            for (int a = 3; a < 6; ++a) s_b[a][threadIdx.x] = fmax(s_b[a][threadIdx.x], s_b[a][threadIdx.x + w]);
        }
        __syncthreads();
    }
    if (threadIdx.x < 6) bbox[blockIdx.x * 6 + threadIdx.x] = s_b[threadIdx.x][0];
    if (threadIdx.x == 0 && s_rej) atomicAdd(rejected, (unsigned long long) s_rej);
}

// step 2: the cell of every valid point, claimed in the table and counted
__global__ void k_count(const double4 *__restrict__ ipts, uint64_t n, GridArgs G, ulonglong2 *table,
                        uint32_t *__restrict__ fill, uint32_t *__restrict__ pslot, unsigned long long *occupied) {
    for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < n; i += (uint64_t) gridDim.x * blockDim.x) {
        const double4 p = ipts[i];
        if (!finite3(p.x, p.y, p.z)) {
            pslot[i] = kNoSlot;
            continue;
        }
        const unsigned long long key = cell_key(cell_of(p.x, G.ox, G.inv, G.nx), cell_of(p.y, G.oy, G.inv, G.ny),
                                                cell_of(p.z, G.oz, G.inv, G.nz));
        uint64_t h = hash_key(key) & G.mask;
        for (;;) {
            const unsigned long long prev = atomicCAS(&table[h].x, kEmptyKey, key);
            if (prev == kEmptyKey) {
                atomicAdd(occupied, 1ull);
                break;
            }
            if (prev == key) break;
            h = (h + 1) & G.mask;
        }
        atomicAdd(fill + h, 1u);
        pslot[i] = (uint32_t) h;
    }
}

// step 3: each occupied cell's range of the cell-ordered array; the cursor of the scatter back to 0
__global__ void k_ranges(ulonglong2 *table, uint64_t cap, uint32_t *__restrict__ fill, unsigned long long *placed) {
    for (uint64_t s = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; s < cap; s += (uint64_t) gridDim.x * blockDim.x) {
        if (table[s].x == kEmptyKey) continue;
        const uint32_t c = fill[s];
        const unsigned long long start = atomicAdd(placed, (unsigned long long) c);
        table[s].y = (start << 32) | c;
        fill[s] = 0;
    }
}

// step 4: the points into their cells' ranges, with their index
__global__ void k_scatter(const double4 *__restrict__ ipts, const uint32_t *__restrict__ pslot, uint64_t n,
                          const ulonglong2 *__restrict__ table, uint32_t *__restrict__ fill, double4 *__restrict__ cpts) {
    for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < n; i += (uint64_t) gridDim.x * blockDim.x) {
        const uint32_t s = pslot[i];
        if (s == kNoSlot) continue;
        const uint64_t pos = (table[s].y >> 32) + atomicAdd(fill + s, 1u);
        const double4 p = ipts[i];
        cpts[pos] = make_double4(p.x, p.y, p.z, __longlong_as_double((long long) i));
    }
}

__device__ __forceinline__ long long point_index(const double4 &p) { return __double_as_longlong(p.w); }
__device__ __forceinline__ void sift_down(double4 *a, uint32_t root, uint32_t end) {
    while (2 * root + 1 < end) {
        uint32_t c = 2 * root + 1;
        if (c + 1 < end && point_index(a[c]) < point_index(a[c + 1])) ++c;
        if (point_index(a[root]) >= point_index(a[c])) return;
        const double4 t = a[root];
        a[root] = a[c];
        a[c] = t;
        root = c;
    }
}
// step 5: each cell's points back into input order (the scatter's order follows the schedule): one thread per cell,
// insertion sort for the small cells the cell size aims at, heap sort for the large cells of duplicate-heavy clouds
__global__ void k_order_cells(const ulonglong2 *__restrict__ table, uint64_t cap, double4 *__restrict__ cpts) {
    for (uint64_t s = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; s < cap; s += (uint64_t) gridDim.x * blockDim.x) {
        const ulonglong2 e = table[s];
        if (e.x == kEmptyKey) continue;
        double4 *a = cpts + (e.y >> 32);
        const uint32_t c = (uint32_t) e.y;
        if (c <= 32) {
            for (uint32_t i = 1; i < c; ++i) {
                const double4 v = a[i];
                uint32_t j = i;
                while (j > 0 && point_index(a[j - 1]) > point_index(v)) {
                    a[j] = a[j - 1];
                    --j;
                }
                a[j] = v;
            }
            continue;
        }
        for (uint32_t r = c / 2; r-- > 0;) sift_down(a, r, c);
        for (uint32_t end = c - 1; end > 0; --end) {
            const double4 t = a[0];
            a[0] = a[end];
            a[end] = t;
            sift_down(a, 0, end);
        }
    }
}

__device__ __forceinline__ double4 ld_point(const double4 *p) {
    const double2 a = __ldg(reinterpret_cast<const double2 *>(p)), b = __ldg(reinterpret_cast<const double2 *>(p) + 1);
    return make_double4(a.x, a.y, b.x, b.y);
}

__device__ __forceinline__ bool probe(const GridArgs &G, unsigned long long key, uint32_t &start, uint32_t &count) {
    uint64_t s = hash_key(key) & G.mask;
    for (;;) {
        const ulonglong2 e = __ldg(G.table + s);
        if (e.x == key) {
            start = (uint32_t) (e.y >> 32);
            count = (uint32_t) e.y;
            return true;
        }
        if (e.x == kEmptyKey) return false;
        s = (s + 1) & G.mask;
    }
}

struct WarpList {
    uint32_t start[kListCap], count[kListCap];
};

// the points of `c` <= 32 staged cells against the held k nearest (all lanes)
__device__ __forceinline__ void consume_cells(const GridArgs &G, const WarpList &L, int c, double qx, double qy,
                                              double qz, double max_radius, int k, int lane, KnnEntry &best,
                                              KnnEntry &kth) {
    const uint32_t ct = lane < c ? L.count[lane] : 0u, st = lane < c ? L.start[lane] : 0u;
    uint32_t incl = ct;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    const uint32_t pre = incl - ct, total = __shfl_sync(0xffffffffu, incl, 31);
    for (uint32_t base = 0; base < total; base += 32) {
        const uint32_t p = base + (uint32_t) lane;
        int lo = 0;   // the last staged cell whose range begins at or before p
#pragma unroll
        for (int step = 16; step > 0; step >>= 1) {
            const uint32_t v = __shfl_sync(0xffffffffu, pre, lo + step);
            if (v <= p) lo += step;
        }
        const uint32_t so = __shfl_sync(0xffffffffu, st, lo), po = __shfl_sync(0xffffffffu, pre, lo);
        KnnEntry cand{INFINITY, 0x7fffffff, 0u};
        bool ok = false;
        if (p < total) {
            const uint32_t pos = so + (p - po);
            const double4 pt = ld_point(G.cpts + pos);
            const double d2 = dist2(qx, qy, qz, pt.x, pt.y, pt.z);
            const KnnEntry e{d2, (int) __double_as_longlong(pt.w), pos};
            if (d2 < max_radius && knn_less(e, kth)) {
                cand = e;
                ok = true;
            }
        }
        if (__ballot_sync(0xffffffffu, ok)) {
            knn_sort32(cand, lane);
            knn_merge32(best, cand, lane);
            kth.d2 = __shfl_sync(0xffffffffu, best.d2, k - 1);
            kth.seq = __shfl_sync(0xffffffffu, best.seq, k - 1);
            kth.addr = __shfl_sync(0xffffffffu, best.addr, k - 1);
        }
    }
}

// the k nearest of query q (valid: finite), held one per lane (lane j: the j-th nearest, d2 = +inf past the count);
// returns the count
__device__ int warp_knn(const GridArgs &G, WarpList &L, double qx, double qy, double qz, int k, double max_radius,
                        int lane, KnnEntry &best) {
    best = KnnEntry{INFINITY, 0x7fffffff, 0u};
    if (G.empty || !finite3(qx, qy, qz) || !(max_radius > 0.0)) return 0;
    KnnEntry kth = best;
    const double lim = 1099511627776.0;   // 2^40 cells: beyond, the ring bounds stay conservative
    const double fx = fmin(fmax((qx - G.ox) * G.inv, -lim), lim), fy = fmin(fmax((qy - G.oy) * G.inv, -lim), lim),
                 fz = fmin(fmax((qz - G.oz) * G.inv, -lim), lim);
    const double flx = floor(fx), fly = floor(fy), flz = floor(fz);
    const long long cx = (long long) flx, cy = (long long) fly, cz = (long long) flz;
    const double gx = fx - flx, gy = fy - fly, gz = fz - flz;
    const double g = fmin(fmin(fmin(gx, 1.0 - gx), fmin(gy, 1.0 - gy)), fmin(gz, 1.0 - gz));
    // the box of cells relative to the query's cell
    const long long lox = -cx, hix = G.nx - 1 - cx, loy = -cy, hiy = G.ny - 1 - cy, loz = -cz, hiz = G.nz - 1 - cz;
    auto out_of = [](long long lo, long long hi) { return lo > 0 ? lo : hi < 0 ? -hi : 0ll; };
    auto reach = [](long long lo, long long hi) { return max(-lo, hi); };
    const long long r0 = max(max(out_of(lox, hix), out_of(loy, hiy)), out_of(loz, hiz));
    const long long r1 = max(max(reach(lox, hix), reach(loy, hiy)), reach(loz, hiz));
    int fill = 0;
    for (long long r = r0; r <= r1; ++r) {
        // every point of ring r and beyond is at least (r - 1 + g) h away (less a margin for the rounding of the cells)
        const double lb = ((double) r - 1.0 + g - 1e-6) * G.h;
        const double lb2 = lb > 0.0 ? lb * lb * (1.0 - 1e-12) : 0.0;
        if (lb2 >= max_radius || (kth.d2 < INFINITY && lb2 > kth.d2)) break;
        const long long x0 = max(-r, lox), x1 = min(r, hix), y0 = max(-r, loy), y1 = min(r, hiy), z0 = max(-r, loz),
                        z1 = min(r, hiz);
        if (x0 > x1 || y0 > y1 || z0 > z1) continue;
        const long long nyr = y1 - y0 + 1, rows = nyr * (z1 - z0 + 1);
        const bool left = -r >= x0, right = r <= x1 && r != 0;
        for (long long t0 = 0; t0 < rows; t0 += 32) {
            const long long t = t0 + lane;
            const bool row = t < rows;
            const long long dz = z0 + (row ? t / nyr : 0), dy = y0 + (row ? t % nyr : 0);
            const bool full = dy == -r || dy == r || dz == -r || dz == r;
            const long long nc = !row ? 0 : full ? x1 - x0 + 1 : (long long) left + (long long) right;
            long long ncmax = nc;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) ncmax = max(ncmax, __shfl_xor_sync(0xffffffffu, ncmax, o));
            for (long long j = 0; j < ncmax; ++j) {
                uint32_t st = 0, ct = 0;
                bool hit = false;
                if (j < nc) {
                    const long long dx = full ? x0 + j : (j == 0 && left) ? -r : r;
                    hit = probe(G, cell_key(cx + dx, cy + dy, cz + dz), st, ct);
                }
                const unsigned m = __ballot_sync(0xffffffffu, hit);
                if (hit) {
                    const int at = fill + __popc(m & ((1u << lane) - 1u));
                    L.start[at] = st;
                    L.count[at] = ct;
                }
                fill += __popc(m);
                __syncwarp();
                if (fill >= 32) {
                    consume_cells(G, L, 32, qx, qy, qz, max_radius, k, lane, best, kth);
                    __syncwarp();
                    if (lane < fill - 32) {
                        L.start[lane] = L.start[32 + lane];
                        L.count[lane] = L.count[32 + lane];
                    }
                    fill -= 32;
                    __syncwarp();
                }
            }
        }
        if (fill) {
            consume_cells(G, L, fill, qx, qy, qz, max_radius, k, lane, best, kth);
            fill = 0;
            __syncwarp();
        }
    }
    return __popc(__ballot_sync(0xffffffffu, lane < k && best.d2 < INFINITY));
}

// ComputeNeighborhood(values) + ClassifyNeighborhood from the moments of n points about the centre c (s: Σ r, then
// Σ r r^T as xx xy xz yy yz zz, r = p - c). The arithmetic of describe_full_from_sums (gather_select.cuh) with the
// reference's divisions. It is restated, not called: that function returns no singular values and a2D needs them
// (from linearity and planarity a2D would lose ~sqrt(u) when sv2 is small), and widening its result would change the
// LM kernel that inlines it.
__device__ __forceinline__ void describe_moments(int n, const double (&s)[9], double cx, double cy, double cz, int values,
                                                double lin_t, double plan_t, cticp_neighborhood_description &d) {
    d.planarity = d.linearity = d.a2D = d.cov_det = -1.0;
    for (int a = 0; a < 3; ++a) d.line[a] = d.normal[a] = d.barycenter[a] = 0.0;
    for (int a = 0; a < 6; ++a) d.covariance[a] = 0.0;
    d.is_valid = 0;
    d.type = CTICP_NB_TYPE_NONE;
    if (n < 5) return;
    const double nn = (double) n;
    const double mx = s[0] / nn, my = s[1] / nn, mz = s[2] / nn;
    double *c = d.covariance;
    c[0] = s[3] / nn - mx * mx;
    c[1] = s[4] / nn - mx * my;
    c[2] = s[5] / nn - mx * mz;
    c[3] = s[6] / nn - my * my;
    c[4] = s[7] / nn - my * mz;
    c[5] = s[8] / nn - mz * mz;
    d.barycenter[0] = cx + mx;
    d.barycenter[1] = cy + my;
    d.barycenter[2] = cz + mz;
    const Eig3Full e = sym_eig3_full(c[0], c[1], c[2], c[3], c[4], c[5]);
    if (values & CTICP_NB_LINE) {
        d.line[0] = e.line.x; d.line[1] = e.line.y; d.line[2] = e.line.z;
    }
    if (values & CTICP_NB_NORMAL) {
        d.normal[0] = e.normal.x; d.normal[1] = e.normal.y; d.normal[2] = e.normal.z;
    }
    if (values & CTICP_NB_LINEARITY) d.linearity = (e.sv0 - e.sv1) / e.sv0;
    if (values & CTICP_NB_PLANARITY) d.planarity = (e.sv1 - e.sv2) / e.sv0;
    if (values & CTICP_NB_A2D) d.a2D = (sqrt(e.sv1) - sqrt(e.sv2)) / sqrt(e.sv0);
    if (values & CTICP_NB_COV_DET) {   // Eigen's determinant of a 3x3: cofactor expansion along the first row
        const double m00 = c[0], m01 = c[1], m02 = c[2], m11 = c[3], m12 = c[4], m22 = c[5];
        const double t0 = __dmul_rn(m00, __dsub_rn(__dmul_rn(m11, m22), __dmul_rn(m12, m12)));
        const double t1 = __dmul_rn(m01, __dsub_rn(__dmul_rn(m01, m22), __dmul_rn(m12, m02)));
        const double t2 = __dmul_rn(m02, __dsub_rn(__dmul_rn(m01, m12), __dmul_rn(m11, m02)));
        d.cov_det = __dadd_rn(__dsub_rn(t0, t1), t2);
    }
    d.is_valid = 1;
    if ((values & CTICP_NB_PLANARITY) && (values & CTICP_NB_LINEARITY)) {
        if (d.planarity > plan_t) d.type = CTICP_NB_TYPE_PLANAR;
        else if (d.linearity > lin_t) d.type = CTICP_NB_TYPE_LINEAR;
    } else if ((values & CTICP_NB_COV_DET) && n > 5) {
        d.type = CTICP_NB_TYPE_VOLUMIC;
    }
}

__device__ __forceinline__ double warp_total(double v) {   // the xor butterfly: every lane ends with the same bits
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

struct QueryArgs {
    const double *queries;   // m xyz triples, or null: the indexed points
    const double4 *ipts;
    uint64_t m;
    int k;
    double max_radius;
    int values;
    double lin_t, plan_t;
    uint64_t *indices;
    double *d2;
    int32_t *counts;
    cticp_neighborhood_description *desc;
};

template <bool DESCRIBE>
__global__ void __launch_bounds__(kThreads, 1) k_query(GridArgs G, QueryArgs Q) {
    __shared__ WarpList s_list[kWarps];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    WarpList &L = s_list[warp];
    for (uint64_t q = blockIdx.x * (uint64_t) kWarps + warp; q < Q.m; q += (uint64_t) gridDim.x * kWarps) {
        double qx, qy, qz;
        if (Q.queries) {
            qx = Q.queries[3 * q]; qy = Q.queries[3 * q + 1]; qz = Q.queries[3 * q + 2];
        } else {
            const double4 p = Q.ipts[q];
            qx = p.x; qy = p.y; qz = p.z;
        }
        KnnEntry best;
        const int n = warp_knn(G, L, qx, qy, qz, Q.k, Q.max_radius, lane, best);
        if (!DESCRIBE) {
            if (lane < Q.k) {
                Q.indices[q * Q.k + lane] = lane < n ? (uint64_t) best.seq : ~0ull;
                Q.d2[q * Q.k + lane] = lane < n ? best.d2 : INFINITY;
            }
            if (lane == 0) Q.counts[q] = n;
            continue;
        }
        double rx = 0.0, ry = 0.0, rz = 0.0;
        if (lane < n) {
            const double4 p = ld_point(G.cpts + best.addr);
            rx = __dsub_rn(p.x, qx); ry = __dsub_rn(p.y, qy); rz = __dsub_rn(p.z, qz);
        }
        double s[9];
        s[0] = warp_total(rx); s[1] = warp_total(ry); s[2] = warp_total(rz);
        s[3] = warp_total(__dmul_rn(rx, rx)); s[4] = warp_total(__dmul_rn(rx, ry)); s[5] = warp_total(__dmul_rn(rx, rz));
        s[6] = warp_total(__dmul_rn(ry, ry)); s[7] = warp_total(__dmul_rn(ry, rz)); s[8] = warp_total(__dmul_rn(rz, rz));
        if (lane == 0) describe_moments(n, s, qx, qy, qz, Q.values, Q.lin_t, Q.plan_t, Q.desc[q]);
    }
}

// one warp per point set: moments about the set's first point, lane-strided, then the butterfly
__global__ void __launch_bounds__(kThreads) k_describe_sets(const double *xyz, const uint64_t *ends, uint64_t num_sets,
                                                            int values, double lin_t, double plan_t,
                                                            cticp_neighborhood_description *out) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint64_t s = blockIdx.x * (uint64_t) kWarps + warp; s < num_sets; s += (uint64_t) gridDim.x * kWarps) {
        const uint64_t b = s ? ends[s - 1] : 0, e = ends[s];
        const double cx = e > b ? xyz[3 * b] : 0.0, cy = e > b ? xyz[3 * b + 1] : 0.0, cz = e > b ? xyz[3 * b + 2] : 0.0;
        double a[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        for (uint64_t i = b + lane; i < e; i += 32) {
            const double rx = __dsub_rn(xyz[3 * i], cx), ry = __dsub_rn(xyz[3 * i + 1], cy), rz = __dsub_rn(xyz[3 * i + 2], cz);
            a[0] = __dadd_rn(a[0], rx); a[1] = __dadd_rn(a[1], ry); a[2] = __dadd_rn(a[2], rz);
            a[3] = __dadd_rn(a[3], __dmul_rn(rx, rx)); a[4] = __dadd_rn(a[4], __dmul_rn(rx, ry));
            a[5] = __dadd_rn(a[5], __dmul_rn(rx, rz)); a[6] = __dadd_rn(a[6], __dmul_rn(ry, ry));
            a[7] = __dadd_rn(a[7], __dmul_rn(ry, rz)); a[8] = __dadd_rn(a[8], __dmul_rn(rz, rz));
        }
#pragma unroll
        for (int v = 0; v < 9; ++v) a[v] = warp_total(a[v]);
        if (lane == 0) {
            const uint64_t cnt = e - b;
            describe_moments(cnt > 0x7fffffffull ? 0x7fffffff : (int) cnt, a, cx, cy, cz, values, lin_t, plan_t, out[s]);
        }
    }
}

}  // namespace

NeighborhoodIndex::NeighborhoodIndex(int device) : device_(device) {
    CT_CUDA_CHECK(cudaSetDevice(device_));
    stream_ = cticp::Stream(cudaStreamNonBlocking);
    ev_in_ = Event(cudaEventDisableTiming);
    ev_out_ = Event(cudaEventDisableTiming);
    cudaStream_t s = stream_.get();
    d_cnt_.reserve(4, s);
    h_cnt_.reserve(4, s);
    d_table_.reserve(64, s);
    table_mask_ = 63;
    CT_CUDA_CHECK(cudaMemsetAsync(d_table_.data(), 0xFF, sizeof(ulonglong2) * 64, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
}

NeighborhoodIndex::~NeighborhoodIndex() {
    if (stream_.get()) {
        cudaSetDevice(device_);
        cudaStreamSynchronize(stream_.get());
    }
}

void NeighborhoodIndex::BuildHost(const double *xyz, uint64_t stride, uint64_t n) {
    if (n && !xyz) throw std::invalid_argument("null xyz");
    if (stride < 24) throw std::invalid_argument("stride_bytes below 24");
    if (n > kMaxPoints) throw std::invalid_argument("more than 2^31 - 1 points");
    CT_CUDA_CHECK(cudaSetDevice(device_));
    cudaStream_t s = stream_.get();
    if (n) {
        const uint64_t bytes = SpanBytes(n, stride, 24, "xyz");
        d_in_.reserve(bytes, s);
        CT_CUDA_CHECK(cudaMemcpyAsync(d_in_.data(), xyz, bytes, cudaMemcpyHostToDevice, s));
        d_ipts_.reserve(n, s);
        d_bbox_.reserve(6 * (uint64_t) Blocks(n), s);
        CT_CUDA_CHECK(cudaMemsetAsync(d_cnt_.data(), 0, sizeof(unsigned long long) * 4, s));
        const bool nat = stride % 8 == 0;
        auto k = nat ? k_load<double, kLoadNatural> : k_load<double, kLoadBytes>;
        k<<<Blocks(n), kThreads, 0, s>>>(d_in_.data(), stride, n, d_ipts_.data(), d_bbox_.data(), d_cnt_.data());
        CT_CUDA_CHECK(cudaGetLastError());
    }
    BuildFromIndexed(n);
}

void NeighborhoodIndex::BuildDevice(const cticp_device_scan &scan, cudaStream_t stream) {
    const uint64_t n = scan.num_points;
    if (scan.xyz_dtype != CTICP_DTYPE_FLOAT32 && scan.xyz_dtype != CTICP_DTYPE_FLOAT64)
        throw std::invalid_argument("x/y/z must be FLOAT32 or FLOAT64");
    if (n && !scan.xyz) throw std::invalid_argument("scan: null xyz");
    if (n > kMaxPoints) throw std::invalid_argument("more than 2^31 - 1 points");
    CT_CUDA_CHECK(cudaSetDevice(device_));
    const uint64_t xsz = scan.xyz_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8;
    if (n) RequireDeviceRange(scan.xyz, SpanBytes(n, scan.xyz_stride_bytes, 3 * xsz, "xyz"), device_, "xyz");
    cudaStream_t s = stream_.get();
    if (n) {
        CT_CUDA_CHECK(cudaEventRecord(ev_in_.get(), stream));
        CT_CUDA_CHECK(cudaStreamWaitEvent(s, ev_in_.get(), 0));
        d_ipts_.reserve(n, s);
        d_bbox_.reserve(6 * (uint64_t) Blocks(n), s);
        CT_CUDA_CHECK(cudaMemsetAsync(d_cnt_.data(), 0, sizeof(unsigned long long) * 4, s));
        const unsigned char *p = static_cast<const unsigned char *>(scan.xyz);
        const bool nat = reinterpret_cast<uintptr_t>(p) % xsz == 0 && scan.xyz_stride_bytes % xsz == 0;
        if (xsz == 8) {
            auto k = nat ? k_load<double, kLoadNatural> : k_load<double, kLoadBytes>;
            k<<<Blocks(n), kThreads, 0, s>>>(p, scan.xyz_stride_bytes, n, d_ipts_.data(), d_bbox_.data(), d_cnt_.data());
        } else {
            auto k = nat ? k_load<float, kLoadNatural> : k_load<float, kLoadBytes>;
            k<<<Blocks(n), kThreads, 0, s>>>(p, scan.xyz_stride_bytes, n, d_ipts_.data(), d_bbox_.data(), d_cnt_.data());
        }
        CT_CUDA_CHECK(cudaGetLastError());
    }
    BuildFromIndexed(n);
}

void NeighborhoodIndex::BuildWorldCloud(WorldCloud &wc) {
    if (wc.Device() != device_) throw std::invalid_argument("the world cloud lives on another device");
    const uint64_t n = wc.NumPoints();
    if (n > kMaxPoints) throw std::invalid_argument("more than 2^31 - 1 points");
    CT_CUDA_CHECK(cudaSetDevice(device_));
    cudaStream_t s = stream_.get();
    if (n) {
        d_in_.reserve(24 * n, s);
        cticp_cloud_sink sink{};
        sink.data = d_in_.data();
        sink.capacity_points = n;
        sink.point_step = 24;
        sink.xyz_dtype = CTICP_DTYPE_FLOAT64;
        sink.world = 1;
        wc.ExportDevice(sink, nullptr, s);   // ordered before what this stream queues next
        d_ipts_.reserve(n, s);
        d_bbox_.reserve(6 * (uint64_t) Blocks(n), s);
        CT_CUDA_CHECK(cudaMemsetAsync(d_cnt_.data(), 0, sizeof(unsigned long long) * 4, s));
        k_load<double, kLoadNatural><<<Blocks(n), kThreads, 0, s>>>(d_in_.data(), 24, n, d_ipts_.data(), d_bbox_.data(),
                                                                     d_cnt_.data());
        CT_CUDA_CHECK(cudaGetLastError());
    }
    BuildFromIndexed(n);
}

void NeighborhoodIndex::Count(double h) {
    cudaStream_t s = stream_.get();
    h_ = h;
    GridArgs G{};
    G.table = d_table_.data();
    G.mask = table_mask_;
    G.ox = lo_[0]; G.oy = lo_[1]; G.oz = lo_[2];
    G.h = h_;
    G.inv = 1.0 / h_;
    G.nx = dims_[0]; G.ny = dims_[1]; G.nz = dims_[2];
    CT_CUDA_CHECK(cudaMemsetAsync(d_table_.data(), 0xFF, sizeof(ulonglong2) * (table_mask_ + 1), s));
    CT_CUDA_CHECK(cudaMemsetAsync(d_fill_.data(), 0, sizeof(uint32_t) * (table_mask_ + 1), s));
    CT_CUDA_CHECK(cudaMemsetAsync(d_cnt_.data() + 1, 0, sizeof(unsigned long long), s));
    k_count<<<Blocks(n_), kThreads, 0, s>>>(d_ipts_.data(), n_, G, d_table_.data(), d_fill_.data(), d_pslot_.data(),
                                            d_cnt_.data() + 1);
    CT_CUDA_CHECK(cudaGetLastError());
    CT_CUDA_CHECK(cudaMemcpyAsync(h_cnt_.data(), d_cnt_.data(), sizeof(unsigned long long) * 2, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    occupied_ = h_cnt_.data()[1];
}

void NeighborhoodIndex::BuildFromIndexed(uint64_t n) {
    cudaStream_t s = stream_.get();
    n_ = n;
    rejected_ = 0;
    occupied_ = 0;
    h_ = 1.0;
    for (int a = 0; a < 3; ++a) {
        lo_[a] = 0.0;
        dims_[a] = 1;
    }
    if (n == 0) return;
    const int nb = Blocks(n);
    h_bbox_.reserve(6 * (uint64_t) nb, s);
    CT_CUDA_CHECK(cudaMemcpyAsync(h_bbox_.data(), d_bbox_.data(), sizeof(double) * 6 * nb, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaMemcpyAsync(h_cnt_.data(), d_cnt_.data(), sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    rejected_ = h_cnt_.data()[0];
    const uint64_t valid = n - rejected_;
    if (valid == 0) return;
    double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int b = 0; b < nb; ++b)
        for (int a = 0; a < 3; ++a) {
            lo[a] = std::min(lo[a], h_bbox_.data()[6 * b + a]);
            hi[a] = std::max(hi[a], h_bbox_.data()[6 * b + 3 + a]);
        }
    double e[3], emax = 0.0;
    for (int a = 0; a < 3; ++a) {
        e[a] = hi[a] - lo[a];
        emax = std::max(emax, e[a]);
        lo_[a] = lo[a];
    }
    if (!std::isfinite(emax)) throw std::invalid_argument("the points span more than the largest double");
    double h0 = 1.0;
    if (emax > 0.0) {
        double v = 1.0;
        for (int a = 0; a < 3; ++a) v *= std::max(e[a], emax * 0x1p-10);
        h0 = std::max(std::cbrt(v * kCellTarget / (double) valid), emax / kMaxCell);
    }
    const uint64_t tcap = Pow2AtLeast(std::max<uint64_t>(2 * valid, 64));
    d_table_.reserve(tcap, s);
    d_fill_.reserve(tcap, s);
    d_pslot_.reserve(n, s);
    d_cpts_.reserve(valid, s);
    table_mask_ = tcap - 1;
    auto set_dims = [&](double h) {
        for (int a = 0; a < 3; ++a) dims_[a] = (int) std::min<double>(std::floor(e[a] / h) + 1.0, kMaxCell + 1.0);
    };
    set_dims(h0);
    Count(h0);
    const double mean = (double) valid / (double) occupied_;
    if (mean > 2.0 * kCellTarget && emax > 0.0) {
        const double h1 = std::max(h0 * std::sqrt(kCellTarget / mean), emax / kMaxCell);
        if (h1 < h0) {
            set_dims(h1);
            Count(h1);
        }
    }
    CT_CUDA_CHECK(cudaMemsetAsync(d_cnt_.data() + 2, 0, sizeof(unsigned long long), s));
    k_ranges<<<Blocks(tcap), kThreads, 0, s>>>(d_table_.data(), tcap, d_fill_.data(), d_cnt_.data() + 2);
    k_scatter<<<Blocks(n), kThreads, 0, s>>>(d_ipts_.data(), d_pslot_.data(), n, d_table_.data(), d_fill_.data(),
                                             d_cpts_.data());
    k_order_cells<<<Blocks(tcap), kThreads, 0, s>>>(d_table_.data(), tcap, d_cpts_.data());
    CT_CUDA_CHECK(cudaGetLastError());
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
}

void NeighborhoodIndex::CheckQuery(const void *queries, uint64_t m, int k, double max_radius) const {
    if (k < 1) throw std::invalid_argument("k must be at least 1");
    if (k > kMaxK) throw UnsupportedError("k above 32");
    if (std::isnan(max_radius)) throw std::invalid_argument("max_radius is NaN");
    if (!queries && m != n_) throw std::invalid_argument("queries NULL (the indexed points): m must be num_points");
    if (m > (1ull << 40)) throw std::invalid_argument("more than 2^40 queries");
}

void NeighborhoodIndex::Enqueue(const double *d_queries, uint64_t m, int k, double max_radius, int values, double lin_t,
                                double plan_t, uint64_t *indices, double *d2, int32_t *counts,
                                cticp_neighborhood_description *out, bool describe) {
    cudaStream_t s = stream_.get();
    if (m == 0) return;
    GridArgs G{};
    G.table = d_table_.data();
    G.mask = table_mask_;
    G.cpts = d_cpts_.data();
    G.ox = lo_[0]; G.oy = lo_[1]; G.oz = lo_[2];
    G.h = h_;
    G.inv = 1.0 / h_;
    G.nx = dims_[0]; G.ny = dims_[1]; G.nz = dims_[2];
    G.empty = occupied_ == 0;
    QueryArgs Q{d_queries, d_ipts_.data(), m, k, max_radius, values, lin_t, plan_t, indices, d2, counts, out};
    if (describe) k_query<true><<<WarpBlocks(m), kThreads, 0, s>>>(G, Q);
    else k_query<false><<<WarpBlocks(m), kThreads, 0, s>>>(G, Q);
    CT_CUDA_CHECK(cudaGetLastError());
}

void NeighborhoodIndex::Search(const double *queries, uint64_t m, int k, double max_radius, uint64_t *indices,
                               double *d2, int32_t *counts) {
    CheckQuery(queries, m, k, max_radius);
    if (m && (!indices || !d2 || !counts)) throw std::invalid_argument("null output");
    CT_CUDA_CHECK(cudaSetDevice(device_));
    cudaStream_t s = stream_.get();
    if (m == 0) return;
    if (queries) {
        d_q_.reserve(3 * m, s);
        CT_CUDA_CHECK(cudaMemcpyAsync(d_q_.data(), queries, sizeof(double) * 3 * m, cudaMemcpyHostToDevice, s));
    }
    d_idx_.reserve(m * k, s);
    d_d2_.reserve(m * k, s);
    d_counts_.reserve(m, s);
    Enqueue(queries ? d_q_.data() : nullptr, m, k, max_radius, 0, 0, 0, d_idx_.data(), d_d2_.data(), d_counts_.data(),
            nullptr, false);
    CT_CUDA_CHECK(cudaMemcpyAsync(indices, d_idx_.data(), sizeof(uint64_t) * m * k, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaMemcpyAsync(d2, d_d2_.data(), sizeof(double) * m * k, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaMemcpyAsync(counts, d_counts_.data(), sizeof(int32_t) * m, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
}

void NeighborhoodIndex::Describe(const double *queries, uint64_t m, int k, double max_radius, int values,
                                 double linearity_threshold, double planarity_threshold,
                                 cticp_neighborhood_description *out) {
    CheckQuery(queries, m, k, max_radius);
    if (m && !out) throw std::invalid_argument("null output");
    CT_CUDA_CHECK(cudaSetDevice(device_));
    cudaStream_t s = stream_.get();
    if (m == 0) return;
    if (queries) {
        d_q_.reserve(3 * m, s);
        CT_CUDA_CHECK(cudaMemcpyAsync(d_q_.data(), queries, sizeof(double) * 3 * m, cudaMemcpyHostToDevice, s));
    }
    d_desc_.reserve(m, s);
    Enqueue(queries ? d_q_.data() : nullptr, m, k, max_radius, values, linearity_threshold, planarity_threshold, nullptr,
            nullptr, nullptr, d_desc_.data(), true);
    CT_CUDA_CHECK(cudaMemcpyAsync(out, d_desc_.data(), sizeof(cticp_neighborhood_description) * m,
                                  cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
}

void NeighborhoodIndex::SearchDevice(const double *queries, uint64_t m, int k, double max_radius, uint64_t *indices,
                                     double *d2, int32_t *counts, cudaStream_t stream) {
    CheckQuery(queries, m, k, max_radius);
    if (m && (!indices || !d2 || !counts)) throw std::invalid_argument("null output");
    CT_CUDA_CHECK(cudaSetDevice(device_));
    if (m == 0) return;
    if (queries) RequireAligned(queries, 8, "queries");
    RequireAligned(indices, 8, "indices");
    RequireAligned(d2, 8, "d2");
    RequireAligned(counts, 4, "counts");
    if (queries) RequireDeviceRange(queries, sizeof(double) * 3 * m, device_, "queries");
    RequireDeviceRange(indices, sizeof(uint64_t) * m * k, device_, "indices");
    RequireDeviceRange(d2, sizeof(double) * m * k, device_, "d2");
    RequireDeviceRange(counts, sizeof(int32_t) * m, device_, "counts");
    cudaStream_t s = stream_.get();
    CT_CUDA_CHECK(cudaEventRecord(ev_in_.get(), stream));
    CT_CUDA_CHECK(cudaStreamWaitEvent(s, ev_in_.get(), 0));
    Enqueue(queries, m, k, max_radius, 0, 0, 0, indices, d2, counts, nullptr, false);
    CT_CUDA_CHECK(cudaEventRecord(ev_out_.get(), s));
    CT_CUDA_CHECK(cudaStreamWaitEvent(stream, ev_out_.get(), 0));
}

void NeighborhoodIndex::DescribeDevice(const double *queries, uint64_t m, int k, double max_radius, int values,
                                       double linearity_threshold, double planarity_threshold,
                                       cticp_neighborhood_description *out, cudaStream_t stream) {
    CheckQuery(queries, m, k, max_radius);
    if (m && !out) throw std::invalid_argument("null output");
    CT_CUDA_CHECK(cudaSetDevice(device_));
    if (m == 0) return;
    if (queries) RequireAligned(queries, 8, "queries");
    RequireAligned(out, 8, "out");
    if (queries) RequireDeviceRange(queries, sizeof(double) * 3 * m, device_, "queries");
    RequireDeviceRange(out, sizeof(cticp_neighborhood_description) * m, device_, "out");
    cudaStream_t s = stream_.get();
    CT_CUDA_CHECK(cudaEventRecord(ev_in_.get(), stream));
    CT_CUDA_CHECK(cudaStreamWaitEvent(s, ev_in_.get(), 0));
    Enqueue(queries, m, k, max_radius, values, linearity_threshold, planarity_threshold, nullptr, nullptr, nullptr, out,
            true);
    CT_CUDA_CHECK(cudaEventRecord(ev_out_.get(), s));
    CT_CUDA_CHECK(cudaStreamWaitEvent(stream, ev_out_.get(), 0));
}

void DescribePointSets(int device, const double *xyz, uint64_t stride, uint64_t n, const uint64_t *segment_ends,
                       uint64_t num_sets, int values, double linearity_threshold, double planarity_threshold,
                       cticp_neighborhood_description *out) {
    if ((n && !xyz) || (num_sets && (!segment_ends || !out))) throw std::invalid_argument("null argument");
    if (stride < 24) throw std::invalid_argument("stride_bytes below 24");
    uint64_t prev = 0;
    for (uint64_t s = 0; s < num_sets; ++s) {
        if (segment_ends[s] < prev || segment_ends[s] > n) throw std::invalid_argument("segment_ends not non-decreasing in [0, n]");
        prev = segment_ends[s];
    }
    if (num_sets && prev != n) throw std::invalid_argument("the last segment end must be n");
    if (num_sets == 0) return;
    CT_CUDA_CHECK(cudaSetDevice(device));
    cticp::Stream stream(cudaStreamNonBlocking);
    cudaStream_t s = stream.get();
    std::vector<double> packed(3 * std::max<uint64_t>(n, 1));
    for (uint64_t i = 0; i < n; ++i) {
        const double *p = reinterpret_cast<const double *>(reinterpret_cast<const unsigned char *>(xyz) + i * stride);
        packed[3 * i] = p[0];
        packed[3 * i + 1] = p[1];
        packed[3 * i + 2] = p[2];
    }
    DeviceArray<double> d_xyz;
    DeviceArray<uint64_t> d_ends;
    DeviceArray<cticp_neighborhood_description> d_out;
    d_xyz.reserve(packed.size(), s);
    d_ends.reserve(num_sets, s);
    d_out.reserve(num_sets, s);
    CT_CUDA_CHECK(cudaMemcpyAsync(d_xyz.data(), packed.data(), sizeof(double) * packed.size(), cudaMemcpyHostToDevice, s));
    CT_CUDA_CHECK(cudaMemcpyAsync(d_ends.data(), segment_ends, sizeof(uint64_t) * num_sets, cudaMemcpyHostToDevice, s));
    k_describe_sets<<<WarpBlocks(num_sets), kThreads, 0, s>>>(d_xyz.data(), d_ends.data(), num_sets, values,
                                                              linearity_threshold, planarity_threshold, d_out.data());
    CT_CUDA_CHECK(cudaGetLastError());
    CT_CUDA_CHECK(cudaMemcpyAsync(out, d_out.data(), sizeof(cticp_neighborhood_description) * num_sets,
                                  cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
}

}  // namespace cticp
