// lidar_sim.cu — a spinning LiDAR ray-cast on the device: ranges of given rays, and sweeps of a sensor moving along a
// continuous trajectory into a host or device sink.
//
// This file is compiled with -fmad=false: every candidate range is the fp64 arithmetic of the host caster
// (tools/raycast.c), operation for operation, so ranges equal the host's bit for bit (porous returns: up to the device
// log's last bit). The host caster tests every primitive against every ray; here the primitives are binned into a
// uniform xy grid when the scene is created (count, ranges, scatter), and a ray walks the cells its xy projection crosses
// (2-D DDA), testing the primitives listed there. The range is the minimum over an order-independent candidate set, so the
// walk may stop once the next cell's entry distance is at least the best candidate found: every primitive is listed in
// each cell its footprint (padded by kPadRel of the scene's scale) touches, and its candidate is never below its entry
// distance. It also stops when the ray has climbed above the tallest primitive or left the grid. It never stops at
// max_range: the host caster prunes by x only, and a box inside that window may be hit beyond it.
// A sweep call runs three steps on the scene's stream:
//   1. the column timestamps, then the trajectory's own k_interpolate at them (on its stream, between two events);
//   2. one pass over tiles of (frame, kThreads rays) in that order, tiles taken from an atomic ticket: each lane casts its
//      ray and applies noise and the keep rule; a tile's kept rays are numbered by a block scan and placed by the
//      decoupled look-back of tile_lookback.cuh, so the output is in (frame, ray) order whatever the schedule;
//   3. the last tile of a frame writes its end.
#include "lidar_sim.h"

#include <algorithm>
#include <cmath>
#include <stdexcept>
#include <string>

#include "device_checks.h"
#include "device_map.h"
#include "record_io.cuh"
#include "se3.cuh"
#include "tile_lookback.cuh"
#include "trajectory.h"

namespace cticp {

namespace {

constexpr int kThreads = 256;
constexpr double kPadRel = 1e-7;               // footprint padding, relative to the scene's largest |coordinate| (>= 1 m)
constexpr uint64_t kMaxCells = 1ull << 22;
constexpr int kMaxCellsPerAxis = 1 << 13;
constexpr uint64_t kNoiseTag = 1ull << 32;     // the frame slot of the noise key (frame ids are 32-bit)

struct SceneArgs {
    const double *boxes;   // nb × 8
    const double4 *cyl;    // nc
    const uint2 *cells;
    const uint32_t *items;
    uint32_t nb;
    int ground;
    LidarGrid G;
};

CT_HD double u01(uint64_t h) { return ((h >> 11) + 0.5) * (1.0 / 9007199254740992.0); }

// a read-only 32-byte load as two 16-byte ones (__ldg has no double4 overload)
__device__ __forceinline__ double4 ldg4(const double4 *p) {
    const double2 a = __ldg(reinterpret_cast<const double2 *>(p)), b = __ldg(reinterpret_cast<const double2 *>(p) + 1);
    return make_double4(a.x, a.y, b.x, b.y);
}

CT_HD bool finite3(double x, double y, double z) { return isfinite(x) && isfinite(y) && isfinite(z); }

// the cells [ix0, ix1] × [iy0, iy1] a footprint [x0, x1] × [y0, y1] padded by pad touches
CT_HD void footprint_cells(const LidarGrid &G, double x0, double y0, double x1, double y1, double pad, int &ix0,
                           int &iy0, int &ix1, int &iy1) {
    ix0 = max(0, min(G.nx - 1, (int) floor((x0 - pad - G.x0) * G.inv_cell)));
    ix1 = max(0, min(G.nx - 1, (int) floor((x1 + pad - G.x0) * G.inv_cell)));
    iy0 = max(0, min(G.ny - 1, (int) floor((y0 - pad - G.y0) * G.inv_cell)));
    iy1 = max(0, min(G.ny - 1, (int) floor((y1 + pad - G.y0) * G.inv_cell)));
}

__device__ __forceinline__ void prim_footprint(const SceneArgs &S, uint32_t id, double pad, int &ix0, int &iy0,
                                               int &ix1, int &iy1) {
    if (id < S.nb) {
        const double *B = S.boxes + 8 * (uint64_t) id;
        footprint_cells(S.G, B[0], B[1], B[3], B[4], pad, ix0, iy0, ix1, iy1);
    } else {
        const double4 c = S.cyl[id - S.nb];
        footprint_cells(S.G, c.x - c.z, c.y - c.z, c.x + c.z, c.y + c.z, pad, ix0, iy0, ix1, iy1);
    }
}

// grid build, step 1: every primitive counted in each cell it touches; the total number of entries
__global__ void __launch_bounds__(kThreads) k_bin_count(SceneArgs S, uint32_t np, double pad, uint32_t *cnt,
                                                        unsigned long long *total) {
    for (uint32_t id = blockIdx.x * blockDim.x + threadIdx.x; id < np; id += gridDim.x * blockDim.x) {
        int ix0, iy0, ix1, iy1;
        prim_footprint(S, id, pad, ix0, iy0, ix1, iy1);
        for (int iy = iy0; iy <= iy1; ++iy)
            for (int ix = ix0; ix <= ix1; ++ix) atomicAdd(&cnt[(uint64_t) iy * S.G.nx + ix], 1u);
        atomicAdd(total, (unsigned long long) (ix1 - ix0 + 1) * (unsigned long long) (iy1 - iy0 + 1));
    }
}

// step 2: each cell's range of the entry array (where it lies follows the schedule); the scatter's cursor back to 0
__global__ void __launch_bounds__(kThreads) k_bin_ranges(uint64_t ncells, uint32_t *cnt, uint2 *cells,
                                                         unsigned long long *placed) {
    for (uint64_t c = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; c < ncells; c += (uint64_t) gridDim.x * blockDim.x) {
        const uint32_t n = cnt[c];
        cells[c] = make_uint2(n ? (uint32_t) atomicAdd(placed, (unsigned long long) n) : 0u, n);
        cnt[c] = 0;
    }
}

// step 3: the primitive ids into their cells' ranges (order within a cell follows the schedule; the range does not)
__global__ void __launch_bounds__(kThreads) k_bin_scatter(SceneArgs S, uint32_t np, double pad, uint32_t *cnt,
                                                          uint32_t *items) {
    for (uint32_t id = blockIdx.x * blockDim.x + threadIdx.x; id < np; id += gridDim.x * blockDim.x) {
        int ix0, iy0, ix1, iy1;
        prim_footprint(S, id, pad, ix0, iy0, ix1, iy1);
        for (int iy = iy0; iy <= iy1; ++iy)
            for (int ix = ix0; ix <= ix1; ++ix) {
                const uint64_t c = (uint64_t) iy * S.G.nx + ix;
                items[S.cells[c].x + atomicAdd(&cnt[c], 1u)] = id;
            }
    }
}

// the candidates of the primitives of one cell, folded into best (tools/raycast.c, operation for operation)
__device__ __forceinline__ void cast_cell(const SceneArgs &S, uint2 range, double ox, double oy, double oz, double dx,
                                          double dy, double dz, double idx, double idy, double idz, double lo, double hi,
                                          double R, uint64_t seed, uint64_t i, double &best) {
    for (uint32_t k = 0; k < range.y; ++k) {
        const uint32_t id = __ldg(S.items + range.x + k);
        if (id < S.nb) {
            const double4 *B4 = reinterpret_cast<const double4 *>(S.boxes + 8 * (uint64_t) id);
            const double4 a = ldg4(B4), b = ldg4(B4 + 1);   // x0 y0 z0 x1 | y1 z1 mfp pad
            if (a.w < lo || a.x > hi) continue;
            double t1 = (a.x - ox) * idx, t2 = (a.w - ox) * idx;
            double tmin = fmin(t1, t2), tmax = fmax(t1, t2);
            t1 = (a.y - oy) * idy;
            t2 = (b.x - oy) * idy;
            tmin = fmax(tmin, fmin(t1, t2));
            tmax = fmin(tmax, fmax(t1, t2));
            t1 = (a.z - oz) * idz;
            t2 = (b.y - oz) * idz;
            tmin = fmax(tmin, fmin(t1, t2));
            tmax = fmin(tmax, fmax(t1, t2));
            if (!(tmax >= tmin) || tmin <= 0 || tmin >= best) continue;
            if (b.z > 0) {
                const double u = u01(splitmix64(seed ^ splitmix64(i * 1315423911ull + id)));
                const double t = tmin - b.z * log(u);
                if (t > tmax || t >= best) continue;
                best = t;
            } else {
                best = tmin;
            }
        } else {
            const double4 C = ldg4(S.cyl + (id - S.nb));   // cx cy r h
            if (fabs(C.x - ox) > R) continue;
            const double px = ox - C.x, py = oy - C.y;
            const double a = dx * dx + dy * dy;
            if (a < 1e-12) continue;
            const double bq = 2 * (px * dx + py * dy), cq = px * px + py * py - C.z * C.z;
            const double disc = bq * bq - 4 * a * cq;
            if (disc <= 0) continue;
            const double t = (-bq - sqrt(disc)) / (2 * a);
            if (t <= 0 || t >= best) continue;
            const double z = oz + t * dz;
            if (z < 0 || z > C.w) continue;
            best = t;
        }
    }
}

// the range of ray i (see include/cticp.h)
__device__ double cast_ray(const SceneArgs &S, double ox, double oy, double oz, double dx, double dy, double dz,
                           double R, uint64_t seed, uint64_t i) {
    if (!finite3(ox, oy, oz) || !finite3(dx, dy, dz)) return __longlong_as_double(0x7ff8000000000000ll);
    double best = INFINITY;
    if (S.ground && dz < 0) {
        const double t = -oz / dz;
        if (t > 0) best = t;
    }
    const LidarGrid &G = S.G;
    if (G.nx == 0) return best;
    const double idx = 1.0 / dx, idy = 1.0 / dy, idz = 1.0 / dz;
    const double lo = ox - R, hi = ox + R;
    // the part of the ray inside the grid's xy box: [tin, tout]
    double tin = 0.0, tout = INFINITY;
    if (dx == 0) {
        if (ox < G.x0 || ox > G.x1) return best;
    } else {
        const double a = (G.x0 - ox) * idx, b = (G.x1 - ox) * idx;
        tin = fmax(tin, fmin(a, b));
        tout = fmin(tout, fmax(a, b));
    }
    if (dy == 0) {
        if (oy < G.y0 || oy > G.y1) return best;
    } else {
        const double a = (G.y0 - oy) * idy, b = (G.y1 - oy) * idy;
        tin = fmax(tin, fmin(a, b));
        tout = fmin(tout, fmax(a, b));
    }
    if (tin > tout) return best;
    int ix = max(0, min(G.nx - 1, (int) floor((ox + tin * dx - G.x0) * G.inv_cell)));
    int iy = max(0, min(G.ny - 1, (int) floor((oy + tin * dy - G.y0) * G.inv_cell)));
    const int sx = dx > 0 ? 1 : -1, sy = dy > 0 ? 1 : -1;
    // the distance at which the ray leaves cell (ix, iy) through its x / y side (INFINITY for no xy motion on that axis)
    auto next_x = [&](int c) { return dx == 0 ? INFINITY : (G.x0 + (double) (c + (dx > 0)) * G.cell - ox) * idx; };
    auto next_y = [&](int c) { return dy == 0 ? INFINITY : (G.y0 + (double) (c + (dy > 0)) * G.cell - oy) * idy; };
    double tx = next_x(ix), ty = next_y(iy);
    for (;;) {
        cast_cell(S, __ldg(S.cells + ((uint64_t) iy * G.nx + ix)), ox, oy, oz, dx, dy, dz, idx, idy, idz, lo, hi, R, seed,
                  i, best);
        const double tn = fmin(tx, ty);
        if (tn >= best || tn > tout) break;                // nothing further can be nearer; or the grid ends
        if (dz > 0 && oz + tn * dz > G.zmax) break;        // above every primitive from here on
        if (tx <= ty) {
            ix += sx;
            if (ix < 0 || ix >= G.nx) break;
            tx = next_x(ix);
        } else {
            iy += sy;
            if (iy < 0 || iy >= G.ny) break;
            ty = next_y(iy);
        }
    }
    return best;
}

__global__ void __launch_bounds__(kThreads) k_raycast(SceneArgs S, const double *__restrict__ o,
                                                      const double *__restrict__ d, uint64_t n, double R, uint64_t seed,
                                                      double *__restrict__ out) {
    for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < n; i += (uint64_t) gridDim.x * blockDim.x)
        out[i] = cast_ray(S, o[3 * i], o[3 * i + 1], o[3 * i + 2], d[3 * i], d[3 * i + 1], d[3 * i + 2], R, seed, i);
}

// the column timestamps t0 + ((j + 0.5) / n_azimuth) period of every frame
__global__ void __launch_bounds__(kThreads) k_column_times(const cticp_lidar_frame *__restrict__ frames, uint64_t m,
                                                           uint32_t naz, double period, double *__restrict__ ts) {
    for (uint64_t k = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; k < m * naz; k += (uint64_t) gridDim.x * blockDim.x) {
        const uint64_t f = k / naz;
        const uint32_t j = (uint32_t) (k - f * naz);
        ts[k] = frames[f].t0 + ((j + 0.5) / naz) * period;
    }
}

// a standard normal of (seed, frame, ray): Box-Muller over two splitmix64 draws
__device__ __forceinline__ double noise_normal(uint64_t seed, uint32_t frame_id, uint64_t i) {
    const uint64_t key = splitmix64(splitmix64(seed) ^ (kNoiseTag | frame_id));
    const double u1 = u01(splitmix64(key ^ (2 * i))), u2 = u01(splitmix64(key ^ (2 * i + 1)));
    return sqrt(-2.0 * log(u1)) * cospi(2.0 * u2);
}

struct SweepArgs {
    const double *cel, *sel, *caz, *saz;     // the direction tables: rings, then columns
    const double *ts;                        // [m naz] column timestamps
    const cticp_pose *poses;                 // [m naz] the poses at them
    const cticp_lidar_frame *frames;
    uint32_t naz;
    uint64_t rays, chunks, tiles;            // per frame; tiles per frame; tiles
    double min_range, max_range, sigma;
    uint64_t seed;
    unsigned long long *desc;                // [tiles] descriptors, [tiles] the ticket
    uint32_t *ray_index;
    uint64_t *ends;
};

// One tile = (frame f, rays [c kThreads, (c + 1) kThreads)); thread j casts ray c kThreads + j.
__global__ void __launch_bounds__(kThreads) k_sweeps(SceneArgs S, SweepArgs g, GenSink sink) {
    __shared__ unsigned long long s_tile;
    __shared__ uint32_t s_warp[kThreads / 32];
    __shared__ uint32_t s_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (;;) {
        if (threadIdx.x == 0) s_tile = atomicAdd(&g.desc[g.tiles], 1ull);
        __syncthreads();
        const unsigned long long tile = s_tile;
        if (tile >= g.tiles) break;
        const uint64_t f = tile / g.chunks, c = tile - f * g.chunks;
        const uint64_t i = c * kThreads + threadIdx.x;
        bool keep = false;
        V3 p{};
        double t = 0.0;
        if (i < g.rays) {
            const uint32_t ring = (uint32_t) (i / g.naz), j = (uint32_t) (i - (uint64_t) ring * g.naz);
            const uint64_t col = f * g.naz + j;
            const cticp_pose &P = g.poses[col];
            const V3 o{P.tr[0], P.tr[1], P.tr[2]};
            const V3 ds{g.cel[ring] * g.caz[j], g.cel[ring] * g.saz[j], g.sel[ring]};
            const V3 dw = qrot(qnormalized(Q4{P.quat[0], P.quat[1], P.quat[2], P.quat[3]}), ds);
            const uint32_t fid = g.frames[f].frame_id;
            double r = cast_ray(S, o.x, o.y, o.z, dw.x, dw.y, dw.z, g.max_range, g.seed * 1000003ull + fid, i);
            if (g.sigma > 0) r = r + g.sigma * noise_normal(g.seed, fid, i);
            keep = isfinite(r) && r > g.min_range && r < g.max_range;
            if (keep) {
                p = sink.world ? V3{o.x + dw.x * r, o.y + dw.y * r, o.z + dw.z * r} : V3{ds.x * r, ds.y * r, ds.z * r};
                t = g.ts[col];
            }
        }
        // block scan of the kept flags: thread order is ray order
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_warp[warp] = __popc(bal);
        __syncthreads();
        uint32_t before = __popc(bal & ((1u << lane) - 1u)), total = 0;
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
        const uint64_t out = (uint64_t) s_base + before;
        if (keep && out < sink.cap) {
            if (sink.data) store_gen_record(sink, out, p, t);
            if (g.ray_index) g.ray_index[out] = (uint32_t) i;
        }
        if (threadIdx.x == 0 && c == g.chunks - 1) g.ends[f] = (uint64_t) s_base + total;
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

void RequireAligned(const void *p, uint64_t align, const char *what) {
    if (reinterpret_cast<uintptr_t>(p) % align)
        throw std::invalid_argument(std::string(what) + " is not " + std::to_string(align) + "-byte aligned");
}

}  // namespace

LidarScene::LidarScene(const double *boxes, uint64_t nb, const double *cylinders, uint64_t nc, bool ground, int device)
    : device_(device), nb_(nb), nc_(nc), ground_(ground) {
    if ((nb && !boxes) || (nc && !cylinders)) throw std::invalid_argument("null primitives");
    if (nb + nc > 0xFFFFFFFFull) throw std::invalid_argument("too many primitives");
    CheckFinite(boxes, 7 * nb, "boxes");
    CheckFinite(cylinders, 4 * nc, "cylinders");
    for (uint64_t b = 0; b < nb; ++b) {
        const double *B = boxes + 7 * b;
        if (B[0] > B[3] || B[1] > B[4] || B[2] > B[5])
            throw std::invalid_argument("box " + std::to_string(b) + ": a lower corner above the upper one");
        if (B[6] < 0) throw std::invalid_argument("box " + std::to_string(b) + ": a negative mean free path");
    }
    for (uint64_t c = 0; c < nc; ++c)
        if (cylinders[4 * c + 2] < 0) throw std::invalid_argument("cylinder " + std::to_string(c) + ": a negative radius");
    // the grid: the primitives' xy box, padded; about one primitive per cell, at most kMaxCells cells
    double x0 = INFINITY, y0 = INFINITY, x1 = -INFINITY, y1 = -INFINITY, zmax = 0.0, scale = 1.0;
    auto grow = [&](double a, double b, double c, double d, double z) {
        x0 = std::min(x0, a);
        y0 = std::min(y0, b);
        x1 = std::max(x1, c);
        y1 = std::max(y1, d);
        zmax = std::max(zmax, z);
        for (double v : {a, b, c, d, z}) scale = std::max(scale, std::fabs(v));
    };
    for (uint64_t b = 0; b < nb; ++b) {
        const double *B = boxes + 7 * b;
        grow(B[0], B[1], B[3], B[4], B[5]);
    }
    for (uint64_t c = 0; c < nc; ++c) {
        const double *C = cylinders + 4 * c;
        grow(C[0] - C[2], C[1] - C[2], C[0] + C[2], C[1] + C[2], C[3]);
    }
    const double pad = kPadRel * scale;
    CT_CUDA_CHECK(cudaSetDevice(device_));
    CT_CUDA_CHECK(cudaDeviceGetAttribute(&sms_, cudaDevAttrMultiProcessorCount, device_));
    CT_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&sweep_ctas_per_sm_, k_sweeps, kThreads, 0));
    sweep_ctas_per_sm_ = std::max(sweep_ctas_per_sm_, 1);
    stream_ = cticp::Stream(cudaStreamNonBlocking);
    ev_in_ = Event(cudaEventDisableTiming);
    ev_traj_ = Event(cudaEventDisableTiming);
    ev_out_ = Event(cudaEventDisableTiming);
    const uint64_t np = nb + nc;
    if (np == 0) return;   // no grid: only the ground
    grid_.x0 = x0 - 2 * pad;
    grid_.y0 = y0 - 2 * pad;
    grid_.x1 = x1 + 2 * pad;
    grid_.y1 = y1 + 2 * pad;
    grid_.zmax = zmax + pad;
    const double w = grid_.x1 - grid_.x0, h = grid_.y1 - grid_.y0;
    double cell = std::max(std::sqrt(w * h / (double) np), std::max(w, h) / kMaxCellsPerAxis);
    while ((uint64_t) std::ceil(w / cell) * (uint64_t) std::ceil(h / cell) > kMaxCells) cell *= 1.25;
    grid_.cell = cell;
    grid_.inv_cell = 1.0 / cell;
    grid_.nx = std::max(1, (int) std::ceil(w / cell));
    grid_.ny = std::max(1, (int) std::ceil(h / cell));
    const uint64_t ncells = NumCells();
    cudaStream_t s = stream_.get();
    std::vector<double> b8(8 * nb, 0.0);
    for (uint64_t b = 0; b < nb; ++b) std::copy(boxes + 7 * b, boxes + 7 * b + 7, b8.begin() + 8 * b);
    d_boxes_.reserve(std::max<uint64_t>(8 * nb, 1), s);
    d_cyl_.reserve(std::max<uint64_t>(4 * nc, 1), s);
    d_cells_.reserve(ncells, s);
    DeviceArray<uint32_t> cnt;
    DeviceArray<unsigned long long> counters;   // [0] entries, [1] the ranges' cursor
    cnt.reserve(ncells, s);
    counters.reserve(2, s);
    if (nb) CT_CUDA_CHECK(cudaMemcpyAsync(d_boxes_.data(), b8.data(), sizeof(double) * 8 * nb, cudaMemcpyHostToDevice, s));
    if (nc) CT_CUDA_CHECK(cudaMemcpyAsync(d_cyl_.data(), cylinders, sizeof(double) * 4 * nc, cudaMemcpyHostToDevice, s));
    CT_CUDA_CHECK(cudaMemsetAsync(cnt.data(), 0, sizeof(uint32_t) * ncells, s));
    CT_CUDA_CHECK(cudaMemsetAsync(counters.data(), 0, sizeof(unsigned long long) * 2, s));
    SceneArgs S{d_boxes_.data(), reinterpret_cast<const double4 *>(d_cyl_.data()), d_cells_.data(), nullptr,
                (uint32_t) nb, ground_ ? 1 : 0, grid_};
    k_bin_count<<<Blocks(np, sms_), kThreads, 0, s>>>(S, (uint32_t) np, pad, cnt.data(), counters.data());
    CT_CUDA_CHECK(cudaGetLastError());
    unsigned long long total = 0;
    CT_CUDA_CHECK(cudaMemcpyAsync(&total, counters.data(), sizeof(total), cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    if (total > 0xFFFFFFFFull) throw CapacityError("the primitives cover more than 2^32 - 1 grid cells in all");
    entries_ = total;
    d_items_.reserve(std::max<uint64_t>(total, 1), s);
    k_bin_ranges<<<Blocks(ncells, sms_), kThreads, 0, s>>>(ncells, cnt.data(), d_cells_.data(), counters.data() + 1);
    k_bin_scatter<<<Blocks(np, sms_), kThreads, 0, s>>>(S, (uint32_t) np, pad, cnt.data(), d_items_.data());
    CT_CUDA_CHECK(cudaGetLastError());
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
}

LidarScene::~LidarScene() {
    if (stream_.get()) {
        cudaSetDevice(device_);
        cudaStreamSynchronize(stream_.get());
    }
}

void LidarScene::LaunchRaycast(const double *o, const double *d, uint64_t n, double max_range, uint64_t seed,
                               double *out) {
    const SceneArgs S{d_boxes_.data(), reinterpret_cast<const double4 *>(d_cyl_.data()), d_cells_.data(),
                      d_items_.data(), (uint32_t) nb_, ground_ ? 1 : 0, grid_};
    k_raycast<<<Blocks(n, sms_), kThreads, 0, stream_.get()>>>(S, o, d, n, max_range, seed, out);
    CT_CUDA_CHECK(cudaGetLastError());
}

void LidarScene::Raycast(const double *origins, const double *directions, uint64_t n, double max_range, uint64_t seed,
                         double *out) {
    if (n && (!origins || !directions || !out)) throw std::invalid_argument("null argument");
    if (!(max_range > 0)) throw std::invalid_argument("max_range must be > 0");
    CheckFinite(origins, 3 * n, "origins");
    CheckFinite(directions, 3 * n, "directions");
    if (n == 0) return;
    CT_CUDA_CHECK(cudaSetDevice(device_));
    cudaStream_t s = stream_.get();
    d_o_.reserve(3 * n, s);
    d_d_.reserve(3 * n, s);
    d_r_.reserve(n, s);
    CT_CUDA_CHECK(cudaMemcpyAsync(d_o_.data(), origins, sizeof(double) * 3 * n, cudaMemcpyHostToDevice, s));
    CT_CUDA_CHECK(cudaMemcpyAsync(d_d_.data(), directions, sizeof(double) * 3 * n, cudaMemcpyHostToDevice, s));
    LaunchRaycast(d_o_.data(), d_d_.data(), n, max_range, seed, d_r_.data());
    CT_CUDA_CHECK(cudaMemcpyAsync(out, d_r_.data(), sizeof(double) * n, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
}

void LidarScene::RaycastDevice(const double *origins, const double *directions, uint64_t n, double max_range,
                               uint64_t seed, double *out, cudaStream_t stream) {
    if (n && (!origins || !directions || !out)) throw std::invalid_argument("null argument");
    if (!(max_range > 0)) throw std::invalid_argument("max_range must be > 0");
    if (n == 0) return;
    CT_CUDA_CHECK(cudaSetDevice(device_));
    RequireAligned(origins, 8, "origins");
    RequireAligned(directions, 8, "directions");
    RequireAligned(out, 8, "out");
    RequireDeviceRange(origins, sizeof(double) * 3 * n, device_, "origins");
    RequireDeviceRange(directions, sizeof(double) * 3 * n, device_, "directions");
    RequireDeviceRange(out, sizeof(double) * n, device_, "out");
    cudaStream_t s = stream_.get();
    CT_CUDA_CHECK(cudaEventRecord(ev_in_.get(), stream));
    CT_CUDA_CHECK(cudaStreamWaitEvent(s, ev_in_.get(), 0));
    LaunchRaycast(origins, directions, n, max_range, seed, out);
    CT_CUDA_CHECK(cudaEventRecord(ev_out_.get(), s));
    CT_CUDA_CHECK(cudaStreamWaitEvent(stream, ev_out_.get(), 0));
}

LidarScene::Plan LidarScene::CheckSweeps(const ContinuousTrajectory &traj, const cticp_lidar_sensor &sensor,
                                         const cticp_lidar_frame *frames, uint64_t m,
                                         const cticp_cloud_sink &sink) const {
    if (m && !frames) throw std::invalid_argument("null frames");
    if (traj.Device() != device_) throw std::invalid_argument("the trajectory lives on another device");
    if (sensor.n_rings == 0 || sensor.n_azimuth == 0) throw std::invalid_argument("n_rings and n_azimuth must be >= 1");
    if (!sensor.elevations_deg) throw std::invalid_argument("null elevations_deg");
    CheckFinite(sensor.elevations_deg, sensor.n_rings, "elevations_deg");
    if (!std::isfinite(sensor.period) || !std::isfinite(sensor.min_range) || !std::isfinite(sensor.max_range))
        throw std::invalid_argument("period, min_range and max_range must be finite");
    if (!(sensor.noise_sigma >= 0) || !std::isfinite(sensor.noise_sigma))
        throw std::invalid_argument("noise_sigma must be finite and >= 0");
    if (!(sensor.max_range > 0)) throw std::invalid_argument("max_range must be > 0");
    for (uint64_t k = 0; k < m; ++k)
        if (!std::isfinite(frames[k].t0)) throw std::invalid_argument("frame " + std::to_string(k) + ": t0 is not finite");
    CheckSink(sink);
    const uint64_t rays = (uint64_t) sensor.n_rings * sensor.n_azimuth;
    if (m && rays > kMaxRays / m) throw CapacityError("more than 2^32 - 1 rays in one call");
    const uint64_t chunks = (rays + kThreads - 1) / kThreads;
    return Plan{m, rays, chunks, m * chunks, m * rays};
}

void LidarScene::Columns(ContinuousTrajectory &traj, const cticp_lidar_sensor &sensor, const cticp_lidar_frame *frames,
                         uint64_t m) {
    cudaStream_t s = stream_.get();
    const uint32_t nr = sensor.n_rings, naz = sensor.n_azimuth;
    std::vector<double> trig(2 * (uint64_t) nr + 2 * (uint64_t) naz);
    for (uint32_t r = 0; r < nr; ++r) {
        const double el = sensor.elevations_deg[r] * (M_PI / 180.0);
        trig[r] = std::cos(el);
        trig[nr + r] = std::sin(el);
    }
    for (uint32_t j = 0; j < naz; ++j) {
        const double az = -2.0 * M_PI * j / naz;
        trig[2 * nr + j] = std::cos(az);
        trig[2 * nr + naz + j] = std::sin(az);
    }
    d_trig_.reserve(trig.size(), s);
    d_frames_.reserve(m, s);
    d_ts_.reserve(m * naz, s);
    d_poses_.reserve(m * naz, s);
    CT_CUDA_CHECK(cudaMemcpyAsync(d_trig_.data(), trig.data(), sizeof(double) * trig.size(), cudaMemcpyHostToDevice, s));
    CT_CUDA_CHECK(cudaMemcpyAsync(d_frames_.data(), frames, sizeof(cticp_lidar_frame) * m, cudaMemcpyHostToDevice, s));
    k_column_times<<<Blocks(m * naz, sms_), kThreads, 0, s>>>(d_frames_.data(), m, naz, sensor.period, d_ts_.data());
    CT_CUDA_CHECK(cudaGetLastError());
    // the trajectory's kernel runs on its own stream, between two events of this one
    CT_CUDA_CHECK(cudaEventRecord(ev_traj_.get(), s));
    CT_CUDA_CHECK(cudaStreamWaitEvent(traj.Stream(), ev_traj_.get(), 0));
    traj.InterpolateDevice(d_ts_.data(), m * naz, d_poses_.data());
    CT_CUDA_CHECK(cudaEventRecord(ev_traj_.get(), traj.Stream()));
    CT_CUDA_CHECK(cudaStreamWaitEvent(s, ev_traj_.get(), 0));
    // the pageable copies above return once `trig` is staged; it may go out of scope
}

void LidarScene::LaunchSweeps(const Plan &plan, const cticp_lidar_sensor &sensor, uint64_t seed,
                              unsigned char *sink_data, const cticp_cloud_sink &sink, uint64_t cap, uint32_t *ray_index,
                              uint64_t *frame_ends) {
    cudaStream_t s = stream_.get();
    d_desc_.reserve(plan.tiles + 1, s);
    CT_CUDA_CHECK(cudaMemsetAsync(d_desc_.data(), 0, sizeof(unsigned long long) * (plan.tiles + 1), s));
    const SceneArgs S{d_boxes_.data(), reinterpret_cast<const double4 *>(d_cyl_.data()), d_cells_.data(),
                      d_items_.data(), (uint32_t) nb_, ground_ ? 1 : 0, grid_};
    const uint32_t nr = sensor.n_rings, naz = sensor.n_azimuth;
    SweepArgs g{};
    g.cel = d_trig_.data();
    g.sel = d_trig_.data() + nr;
    g.caz = d_trig_.data() + 2 * nr;
    g.saz = d_trig_.data() + 2 * nr + naz;
    g.ts = d_ts_.data();
    g.poses = d_poses_.data();
    g.frames = d_frames_.data();
    g.naz = naz;
    g.rays = plan.rays;
    g.chunks = plan.chunks;
    g.tiles = plan.tiles;
    g.min_range = sensor.min_range;
    g.max_range = sensor.max_range;
    g.sigma = sensor.noise_sigma;
    g.seed = seed;
    g.desc = d_desc_.data();
    g.ray_index = ray_index;
    g.ends = frame_ends;
    // as many CTAs as are resident at once (tiles are handed out by the ticket, so any grid size is correct)
    const int blocks = (int) std::min<uint64_t>(plan.tiles, (uint64_t) sms_ * sweep_ctas_per_sm_);
    k_sweeps<<<blocks, kThreads, 0, s>>>(S, g, MakeGenSink(sink_data, sink, cap));
    CT_CUDA_CHECK(cudaGetLastError());
}

int64_t LidarScene::GenerateSweeps(ContinuousTrajectory &traj, const cticp_lidar_sensor &sensor,
                                   const cticp_lidar_frame *frames, uint64_t m, uint64_t seed,
                                   const cticp_cloud_sink &sink, uint32_t *ray_index, uint64_t *frame_ends) {
    if (m && !frame_ends) throw std::invalid_argument("null frame_ends");
    const Plan plan = CheckSweeps(traj, sensor, frames, m, sink);
    if (m == 0) return 0;
    const uint64_t cap = std::min<uint64_t>(sink.data || ray_index ? sink.capacity_points : 0, plan.upper);
    const uint64_t out_bytes = sink.data && cap ? SpanBytes(cap, sink.point_step, SinkRecordWidth(sink), "sink") : 0;
    CT_CUDA_CHECK(cudaSetDevice(device_));
    cudaStream_t s = stream_.get();
    d_out_.reserve(std::max<uint64_t>(out_bytes, 1), s);
    d_idx_.reserve(std::max<uint64_t>(cap, 1), s);
    d_ends_.reserve(m, s);
    // the sink goes over as it is: its bytes outside x, y, z and t stay the caller's
    if (out_bytes) CT_CUDA_CHECK(cudaMemcpyAsync(d_out_.data(), sink.data, out_bytes, cudaMemcpyHostToDevice, s));
    Columns(traj, sensor, frames, m);
    LaunchSweeps(plan, sensor, seed, out_bytes ? d_out_.data() : nullptr, sink, cap, ray_index ? d_idx_.data() : nullptr,
                 d_ends_.data());
    CT_CUDA_CHECK(cudaMemcpyAsync(frame_ends, d_ends_.data(), sizeof(uint64_t) * m, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    const uint64_t count = frame_ends[m - 1], w = std::min(cap, count);
    if (w && out_bytes)
        CT_CUDA_CHECK(cudaMemcpyAsync(sink.data, d_out_.data(), SpanBytes(w, sink.point_step, SinkRecordWidth(sink), "sink"),
                                      cudaMemcpyDeviceToHost, s));
    if (w && ray_index)
        CT_CUDA_CHECK(cudaMemcpyAsync(ray_index, d_idx_.data(), sizeof(uint32_t) * w, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    return (int64_t) count;
}

void LidarScene::GenerateSweepsDevice(ContinuousTrajectory &traj, const cticp_lidar_sensor &sensor,
                                      const cticp_lidar_frame *frames, uint64_t m, uint64_t seed,
                                      const cticp_cloud_sink &sink, uint32_t *ray_index, uint64_t *frame_ends,
                                      cudaStream_t stream) {
    if (m && !frame_ends) throw std::invalid_argument("null frame_ends");
    const Plan plan = CheckSweeps(traj, sensor, frames, m, sink);
    if (m == 0) return;
    const uint64_t cap = std::min<uint64_t>(sink.data || ray_index ? sink.capacity_points : 0, plan.upper);
    CT_CUDA_CHECK(cudaSetDevice(device_));
    RequireAligned(frame_ends, 8, "frame_ends");
    RequireDeviceRange(frame_ends, sizeof(uint64_t) * m, device_, "frame_ends");
    if (ray_index && cap) {
        RequireAligned(ray_index, 4, "ray_index");
        RequireDeviceRange(ray_index, sizeof(uint32_t) * cap, device_, "ray_index");
    }
    if (sink.data && cap)
        RequireDeviceRange(sink.data, SpanBytes(cap, sink.point_step, SinkRecordWidth(sink), "sink"), device_, "sink");
    cudaStream_t s = stream_.get();
    // ordered both ways with the caller's stream: behind what it queued before, ahead of what it queues next
    CT_CUDA_CHECK(cudaEventRecord(ev_in_.get(), stream));
    CT_CUDA_CHECK(cudaStreamWaitEvent(s, ev_in_.get(), 0));
    Columns(traj, sensor, frames, m);
    LaunchSweeps(plan, sensor, seed, sink.data && cap ? static_cast<unsigned char *>(sink.data) : nullptr, sink, cap,
                 ray_index && cap ? ray_index : nullptr, frame_ends);
    CT_CUDA_CHECK(cudaEventRecord(ev_out_.get(), s));
    CT_CUDA_CHECK(cudaStreamWaitEvent(stream, ev_out_.get(), 0));
}

}  // namespace cticp
