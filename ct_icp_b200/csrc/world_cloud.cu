// world_cloud.cu — slam::SamplePointsInGrid (include/SlamCore/algorithm/grid_sampling.h:48-79) and its incremental form.
//
// The reference keeps, per voxel (slam::Voxel::Coordinates: int(p / grid_size), truncation), the first
// num_points_per_voxel points in input order, the first one always. A cloud holds that state on the device for
// every point submitted so far: a committed hash table {voxel key → voxel id}, voxel ids in order of first appearance,
// and per voxel up to kp pool indices in input order. One add of m points runs
//   1. k_key: read (and, for the trajectory / odometry inputs, the world points the trajectory's or the odometry's own
//      kernels wrote), key, look the voxel up in the committed table (read-only) or claim it in a call-local table whose
//      entry keeps the smallest point index (atomicMin): the voxel's first appearance in this call;
//   2. k_first_flags + a scan: new voxels numbered in order of first appearance;
//   3. kp rounds of k_cand / k_take: round r gives each voxel that still has a free slot the smallest point index above
//      the one taken in round r - 1, so the points kept are the smallest indices, whatever the schedule;
//   4. a scan of the kept flags (pool offsets), the capacity check on the host, then k_commit_voxels / k_commit.
// Nothing persistent is written before step 4 except the rank scratch of committed voxels, which step 4 or the refusal
// path puts back. Every result depends on the input order only: run to run, the cloud is bit-identical.
#include "world_cloud.h"

#include <algorithm>
#include <cmath>
#include <limits>
#include <stdexcept>
#include <string>
#include <vector>

#include "device_checks.h"
#include "device_map.cuh"
#include "device_map.h"
#include "engine.h"
#include "record_io.cuh"
#include "scan_pack.cuh"
#include "tile_lookback.cuh"
#include "trajectory.h"

namespace cticp {

namespace {

constexpr int kThreads = 256;
constexpr int kScanItems = 8;                           // per thread: tiles of 2048
constexpr int kScanTile = kThreads * kScanItems;
constexpr uint32_t kRejected = 0xFFFFFFFFu;
constexpr uint32_t kLocal = 0x80000000u;                // pv: a voxel of the call-local table (slot in the low bits)
constexpr uint64_t kMaxCallPoints = 1ull << 30;

int Blocks(uint64_t n) { return (int) std::max<uint64_t>(1, std::min<uint64_t>((n + kThreads - 1) / kThreads, 132 * 16)); }

uint64_t Pow2AtLeast(uint64_t n) {
    uint64_t p = 1;
    while (p < n) p <<= 1;
    return p;
}

struct KeyArgs {
    double res, inv;
    const ulonglong2 *table;   // committed, read-only during the call
    uint64_t table_mask;
    ulonglong2 *ltab;          // call-local
    uint64_t ltab_mask;
};

// step 1. Reads record i (x, y, z of XT, a timestamp of t_dtype or none), writes (x, y, z, t) in fp64 to w[i] and the
// voxel of the point to pv[i]: a committed voxel id, kLocal | call-local slot, or kRejected.
// (xyz / t may be w itself: each thread reads its record before it writes it)
template <typename XT, int LOAD>
__global__ void __launch_bounds__(kThreads) k_key(const unsigned char *xyz, size_t xs, const unsigned char *t, size_t ts,
                                                  int t_dtype, int t_aligned, uint64_t m, KeyArgs A, double4 *w,
                                                  uint32_t *__restrict__ pv, unsigned long long *__restrict__ rejected) {
    for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < m; i += (uint64_t) gridDim.x * blockDim.x) {
        XT x, y, z;
        if (LOAD == kLoadVec4 && i == m - 1)   // the last record read: 12 bytes (a 16-byte load may pass the buffer)
            load_xyz<XT, kLoadNatural>(xyz + i * xs, x, y, z);
        else
            load_xyz<XT, LOAD>(xyz + i * xs, x, y, z);
        const double tt = t_dtype ? load_timestamp(t + i * ts, t_dtype, t_aligned) : 0.0;
        const double px = (double) x, py = (double) y, pz = (double) z;
        w[i] = make_double4(px, py, pz, tt);
        unsigned long long key;
        if (!voxel_key(px, py, pz, A.res, A.inv, key)) {
            pv[i] = kRejected;
            atomicAdd(rejected, 1ull);
            continue;
        }
        uint64_t h = hash_key(key) & A.table_mask;
        uint32_t found = kRejected;
        for (;;) {
            const ulonglong2 s = A.table[h];
            if (s.x == key) {
                found = (uint32_t) s.y;
                break;
            }
            if (s.x == kEmptyKey) break;
            h = (h + 1) & A.table_mask;
        }
        if (found != kRejected) {
            pv[i] = found;
            continue;
        }
        h = hash_key(key) & A.ltab_mask;
        for (;;) {
            const unsigned long long prev = atomicCAS(&A.ltab[h].x, kEmptyKey, key);
            if (prev == kEmptyKey || prev == key) break;
            h = (h + 1) & A.ltab_mask;
        }
        atomicMin(&A.ltab[h].y, (unsigned long long) i);
        pv[i] = kLocal | (uint32_t) h;
    }
}

// step 2: flag[first point of each new voxel] = 1
__global__ void k_first_flags(const ulonglong2 *__restrict__ ltab, uint64_t n, uint32_t *__restrict__ flag) {
    for (uint64_t s = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; s < n; s += (uint64_t) gridDim.x * blockDim.x) {
        const ulonglong2 e = ltab[s];
        if (e.x != kEmptyKey) flag[e.y] = 1u;
    }
}

// pv of the points of new voxels: cap_v + the voxel's rank among the new voxels (first appearance)
__global__ void k_resolve(const ulonglong2 *__restrict__ ltab, const uint32_t *__restrict__ first_rank, uint64_t m,
                          uint32_t cap_v, uint32_t *__restrict__ pv) {
    for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < m; i += (uint64_t) gridDim.x * blockDim.x) {
        const uint32_t v = pv[i];
        if (v != kRejected && (v & kLocal)) pv[i] = cap_v + first_rank[ltab[v & ~kLocal].y];
    }
}

struct RankArgs {
    const uint32_t *vcount;   // committed voxels: points held before this call
    uint32_t *vlo, *vcand;    // committed voxels' rank scratch
    uint32_t *nlo, *ncand;    // new voxels' (index pv - cap_v)
    uint32_t cap_v;
    int kp;
};
__device__ __forceinline__ void rank_refs(const RankArgs &R, uint32_t v, uint32_t &c0, uint32_t *&lo, uint32_t *&cand) {
    if (v < R.cap_v) {
        c0 = __ldg(R.vcount + v);
        lo = R.vlo + v;
        cand = R.vcand + v;
    } else {
        c0 = 0;
        lo = R.nlo + (v - R.cap_v);
        cand = R.ncand + (v - R.cap_v);
    }
}

// step 3, round r: the smallest point index not yet taken of every voxel with a free slot
__global__ void k_cand(const uint32_t *__restrict__ pv, uint64_t m, RankArgs R, int r) {
    for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < m; i += (uint64_t) gridDim.x * blockDim.x) {
        const uint32_t v = pv[i];
        if (v == kRejected) continue;
        uint32_t c0, *lo, *cand;
        rank_refs(R, v, c0, lo, cand);
        if (c0 + (uint32_t) r >= (uint32_t) R.kp || (uint32_t) i < *lo) continue;
        atomicMin(cand, (uint32_t) i);
    }
}
// the candidate takes slot c0 + r (slot[i] = that + 1) and keep[i] = 1; its voxel's next round starts above it
__global__ void k_take(const uint32_t *__restrict__ pv, uint64_t m, RankArgs R, int r, uint32_t *__restrict__ slot,
                       uint32_t *__restrict__ keep) {
    for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < m; i += (uint64_t) gridDim.x * blockDim.x) {
        const uint32_t v = pv[i];
        if (v == kRejected) continue;
        uint32_t c0, *lo, *cand;
        rank_refs(R, v, c0, lo, cand);
        if (*cand != (uint32_t) i) continue;   // one point per voxel matches
        slot[i] = c0 + (uint32_t) r + 1u;
        keep[i] = 1u;
        *lo = (uint32_t) i + 1u;
        *cand = 0xFFFFFFFFu;
    }
}

// the rank scratch of committed voxels back to its resting state (commit and refusal)
__global__ void k_reset_lo(const uint32_t *__restrict__ pv, uint64_t m, uint32_t cap_v, uint32_t *__restrict__ vlo) {
    for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < m; i += (uint64_t) gridDim.x * blockDim.x) {
        const uint32_t v = pv[i];
        if (v != kRejected && v < cap_v) vlo[v] = 0u;
    }
}

// step 4: the new voxels into the committed table, with ids num_voxels + rank
__global__ void k_commit_voxels(const ulonglong2 *__restrict__ ltab, uint64_t n, const uint32_t *__restrict__ first_rank,
                                uint64_t num_voxels, ulonglong2 *__restrict__ table, uint64_t table_mask) {
    for (uint64_t s = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; s < n; s += (uint64_t) gridDim.x * blockDim.x) {
        const ulonglong2 e = ltab[s];
        if (e.x == kEmptyKey) continue;
        uint64_t h = hash_key(e.x) & table_mask;
        while (atomicCAS(&table[h].x, kEmptyKey, e.x) != kEmptyKey) h = (h + 1) & table_mask;
        table[h].y = num_voxels + first_rank[e.y];
    }
}
// the kept points into the pool, in input order, and into their voxels' slots
__global__ void k_commit(const uint32_t *__restrict__ pv, const uint32_t *__restrict__ slot,
                         const uint32_t *__restrict__ pool_off, const double4 *__restrict__ w, uint64_t m, uint32_t cap_v,
                         uint64_t num_voxels, uint64_t num_points, uint64_t num_submitted, int kp,
                         uint32_t *__restrict__ vcount, uint32_t *__restrict__ vpts, double4 *__restrict__ pxyzt,
                         uint64_t *__restrict__ psrc) {
    for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < m; i += (uint64_t) gridDim.x * blockDim.x) {
        const uint32_t s = slot[i];
        if (!s) continue;
        const uint32_t v = pv[i];
        const uint64_t vid = v < cap_v ? (uint64_t) v : num_voxels + (v - cap_v);
        const uint64_t p = num_points + pool_off[i];
        pxyzt[p] = w[i];
        psrc[p] = num_submitted + i;
        vpts[vid * kp + (s - 1u)] = (uint32_t) p;
        atomicMax(vcount + vid, s);
    }
}

// exclusive scan of n counts, tiles taken in launch order from a ticket (tile_lookback.cuh); total: the sum
__global__ void __launch_bounds__(kThreads) k_scan(const uint32_t *__restrict__ in, uint32_t *__restrict__ out, uint64_t n,
                                                   unsigned long long *desc, uint32_t *ticket,
                                                   unsigned long long *total) {
    __shared__ uint32_t s_tile, s_warp[kThreads / 32], s_before;
    if (threadIdx.x == 0) s_tile = atomicAdd(ticket, 1u);
    __syncthreads();
    const uint32_t tile = s_tile;
    const uint64_t base = (uint64_t) tile * kScanTile + (uint64_t) threadIdx.x * kScanItems;
    uint32_t v[kScanItems], sum = 0;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
        v[k] = base + k < n ? in[base + k] : 0u;
        sum += v[k];
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t o = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += o;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint32_t wv = lane < kThreads / 32 ? s_warp[lane] : 0u, wi = wv;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t o = __shfl_up_sync(0xffffffffu, wi, d);
            if (lane >= d) wi += o;
        }
        const uint32_t tile_sum = __shfl_sync(0xffffffffu, wi, 31);
        const uint32_t before = tile_lookback(desc, (int) tile, tile_sum);
        if (lane < kThreads / 32) s_warp[lane] = wi - wv;
        if (lane == 0) {
            s_before = before;
            if ((uint64_t) (tile + 1) * kScanTile >= n) *total = (unsigned long long) before + tile_sum;
        }
    }
    __syncthreads();
    uint32_t run = s_before + s_warp[warp] + incl - sum;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
        if (base + k < n) out[base + k] = run;
        run += v[k];
    }
}

struct SinkArgs {
    unsigned char *data;
    uint32_t step, xoff, toff;
    int xdt, tdt, x_aligned, t_aligned;
};

// voxel-major export: voxel v's points at off[v] onwards, in input order; only positions below lim are written
__global__ void k_export(const uint32_t *__restrict__ vcount, const uint32_t *__restrict__ off,
                         const uint32_t *__restrict__ vpts, const double4 *__restrict__ pxyzt,
                         const uint64_t *__restrict__ psrc, uint64_t num_voxels, int kp, uint64_t lim, SinkArgs sink,
                         uint64_t *__restrict__ src_out) {
    for (uint64_t v = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; v < num_voxels; v += (uint64_t) gridDim.x * blockDim.x) {
        const uint32_t c = vcount[v];
        const uint64_t o = off[v];
        for (uint32_t j = 0; j < c && o + j < lim; ++j) {
            const uint32_t p = vpts[v * kp + j];
            const double4 q = pxyzt[p];
            if (sink.data) {
                unsigned char *rec = sink.data + (o + j) * sink.step;
                if (sink.xdt == CTICP_DTYPE_FLOAT32) {
                    store_field<float>(rec + sink.xoff, scan_pack::hi_of(q.x), sink.x_aligned);
                    store_field<float>(rec + sink.xoff + 4, scan_pack::hi_of(q.y), sink.x_aligned);
                    store_field<float>(rec + sink.xoff + 8, scan_pack::hi_of(q.z), sink.x_aligned);
                } else {
                    store_field<double>(rec + sink.xoff, q.x, sink.x_aligned);
                    store_field<double>(rec + sink.xoff + 8, q.y, sink.x_aligned);
                    store_field<double>(rec + sink.xoff + 16, q.z, sink.x_aligned);
                }
                if (sink.tdt == CTICP_DTYPE_FLOAT32) store_field<float>(rec + sink.toff, scan_pack::hi_of(q.w), sink.t_aligned);
                else if (sink.tdt == CTICP_DTYPE_FLOAT64) store_field<double>(rec + sink.toff, q.w, sink.t_aligned);
            }
            if (src_out) src_out[o + j] = psrc[p];
        }
    }
}

void CheckRecordDtypes(int xyz_dtype, int t_dtype, bool need_t) {
    if (xyz_dtype != CTICP_DTYPE_FLOAT32 && xyz_dtype != CTICP_DTYPE_FLOAT64)
        throw std::invalid_argument("x/y/z must be FLOAT32 or FLOAT64");
    if (t_dtype == 0) {
        if (need_t) throw std::invalid_argument("a trajectory needs the timestamps (t_dtype 0 = none)");
        return;
    }
    if (!scan_pack::dtype_size(t_dtype)) throw std::invalid_argument("unknown timestamp dtype");
}

// the records the trajectory writes and the key pass reads back: x, y, z, t in fp64
cticp_cloud_sink WorldSink(double4 *d, uint64_t m) {
    cticp_cloud_sink s{};
    s.data = d;
    s.capacity_points = m;
    s.point_step = sizeof(double4);
    s.xyz_offset = 0;
    s.xyz_dtype = CTICP_DTYPE_FLOAT64;
    s.t_offset = 24;
    s.t_dtype = CTICP_DTYPE_FLOAT64;
    s.world = 1;
    return s;
}

}  // namespace

void WorldCloud::CheckOptions(const cticp_grid_sampling_options &o) {
    if (!(std::isfinite(o.grid_size) && o.grid_size > 0.0)) throw std::invalid_argument("grid_size must be finite and > 0");
    if (o.num_points_per_voxel < 0 || o.num_points_per_voxel > kMaxPointsPerVoxel)
        throw UnsupportedError("num_points_per_voxel outside [0, 64]");
}

void DefaultCapacity(const cticp_grid_sampling_options &o, uint64_t *capacity_voxels, uint64_t *capacity_points) {
    const double r = 0.2 / o.grid_size;
    const double v = std::min(std::max(4194304.0 * r * r, 65536.0), 67108864.0);
    const uint64_t kp = (uint64_t) std::max(1, o.num_points_per_voxel);
    if (*capacity_voxels == 0) *capacity_voxels = (uint64_t) v;
    if (*capacity_points == 0) *capacity_points = std::min<uint64_t>(*capacity_voxels * kp, 0xFFFFFFFFull);
}

WorldCloud::WorldCloud(const cticp_grid_sampling_options &o, uint64_t capacity_voxels, uint64_t capacity_points,
                       int device)
    : opt_(o), device_(device) {
    CheckOptions(o);
    DefaultCapacity(o, &capacity_voxels, &capacity_points);
    if (capacity_voxels > (1ull << 30)) throw std::invalid_argument("capacity_voxels above 2^30");
    if (capacity_points > 0xFFFFFFFFull) throw std::invalid_argument("capacity_points above 2^32 - 1");
    kp_ = std::max(1, o.num_points_per_voxel);
    cap_v_ = capacity_voxels;
    cap_p_ = capacity_points;
    const uint64_t tcap = Pow2AtLeast(std::max<uint64_t>(2 * cap_v_, 64));
    table_mask_ = tcap - 1;
    CT_CUDA_CHECK(cudaSetDevice(device_));
    stream_ = cticp::Stream(cudaStreamNonBlocking);
    ev_in_ = Event(cudaEventDisableTiming);
    ev_out_ = Event(cudaEventDisableTiming);
    cudaStream_t s = stream_.get();
    d_table_.reserve(tcap, s);
    d_vcount_.reserve(std::max<uint64_t>(cap_v_, 1), s);
    d_vpts_.reserve(std::max<uint64_t>(cap_v_ * kp_, 1), s);
    d_vlo_.reserve(std::max<uint64_t>(cap_v_, 1), s);
    d_vcand_.reserve(std::max<uint64_t>(cap_v_, 1), s);
    d_off_.reserve(std::max<uint64_t>(cap_v_, 1), s);
    d_pxyzt_.reserve(std::max<uint64_t>(cap_p_, 1), s);
    d_psrc_.reserve(std::max<uint64_t>(cap_p_, 1), s);
    d_cnt_.reserve(4, s);
    h_cnt_.reserve(4, s);
    d_ticket_.reserve(1, s);
    CT_CUDA_CHECK(cudaMemsetAsync(d_vlo_.data(), 0, sizeof(uint32_t) * std::max<uint64_t>(cap_v_, 1), s));
    CT_CUDA_CHECK(cudaMemsetAsync(d_vcand_.data(), 0xFF, sizeof(uint32_t) * std::max<uint64_t>(cap_v_, 1), s));
    Clear();
}

WorldCloud::~WorldCloud() {
    if (stream_.get()) {
        cudaSetDevice(device_);
        cudaStreamSynchronize(stream_.get());
    }
}

uint64_t WorldCloud::NumPoints() const {
    if (opt_.max_num_points < 0) return num_points_;
    return std::min<uint64_t>(num_points_, (uint64_t) opt_.max_num_points + 1);
}

void WorldCloud::Clear() {
    CT_CUDA_CHECK(cudaSetDevice(device_));
    cudaStream_t s = stream_.get();
    CT_CUDA_CHECK(cudaMemsetAsync(d_table_.data(), 0xFF, sizeof(ulonglong2) * (table_mask_ + 1), s));
    CT_CUDA_CHECK(cudaMemsetAsync(d_vcount_.data(), 0, sizeof(uint32_t) * std::max<uint64_t>(cap_v_, 1), s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    num_voxels_ = num_points_ = num_submitted_ = 0;
}

void WorldCloud::Scan(const uint32_t *in, uint32_t *out, uint64_t n, int counter) {
    cudaStream_t s = stream_.get();
    const uint64_t tiles = std::max<uint64_t>(1, (n + kScanTile - 1) / kScanTile);
    d_desc_.reserve(tiles, s);
    CT_CUDA_CHECK(cudaMemsetAsync(d_desc_.data(), 0, sizeof(unsigned long long) * tiles, s));
    CT_CUDA_CHECK(cudaMemsetAsync(d_ticket_.data(), 0, sizeof(uint32_t), s));
    CT_CUDA_CHECK(cudaMemsetAsync(d_cnt_.data() + counter, 0, sizeof(unsigned long long), s));
    k_scan<<<(unsigned) tiles, kThreads, 0, s>>>(in, out, n, d_desc_.data(), d_ticket_.data(), d_cnt_.data() + counter);
    CT_CUDA_CHECK(cudaGetLastError());
}

void WorldCloud::Ingest(const unsigned char *xyz, size_t xs, int xyz_dtype, const unsigned char *t, size_t ts, int t_dtype,
                        uint64_t m, cticp_world_cloud_stats *stats) {
    cudaStream_t s = stream_.get();
    cticp_world_cloud_stats st{};
    st.submitted = m;
    if (m == 0) {
        if (stats) *stats = st;
        return;
    }
    const uint64_t lcap = Pow2AtLeast(std::max<uint64_t>(2 * m, 64));
    d_w_.reserve(m, s);
    for (auto *a : {&d_pv_, &d_slot_, &d_flag_, &d_keep_, &d_scan0_, &d_scan1_, &d_nlo_, &d_ncand_}) a->reserve(m, s);
    d_ltab_.reserve(lcap, s);
    CT_CUDA_CHECK(cudaMemsetAsync(d_ltab_.data(), 0xFF, sizeof(ulonglong2) * lcap, s));
    CT_CUDA_CHECK(cudaMemsetAsync(d_flag_.data(), 0, sizeof(uint32_t) * m, s));
    CT_CUDA_CHECK(cudaMemsetAsync(d_keep_.data(), 0, sizeof(uint32_t) * m, s));
    CT_CUDA_CHECK(cudaMemsetAsync(d_slot_.data(), 0, sizeof(uint32_t) * m, s));
    CT_CUDA_CHECK(cudaMemsetAsync(d_nlo_.data(), 0, sizeof(uint32_t) * m, s));
    CT_CUDA_CHECK(cudaMemsetAsync(d_ncand_.data(), 0xFF, sizeof(uint32_t) * m, s));
    CT_CUDA_CHECK(cudaMemsetAsync(d_cnt_.data(), 0, sizeof(unsigned long long) * 4, s));
    KeyArgs A;
    A.res = opt_.grid_size;
    A.inv = 1.0 / opt_.grid_size;
    A.table = d_table_.data();
    A.table_mask = table_mask_;
    A.ltab = d_ltab_.data();
    A.ltab_mask = lcap - 1;
    const size_t xsz = xyz_dtype == CTICP_DTYPE_FLOAT64 ? 8 : 4, tsz = t_dtype ? scan_pack::dtype_size(t_dtype) : 1;
    const bool x_nat = (reinterpret_cast<uintptr_t>(xyz) % xsz) == 0 && xs % xsz == 0;
    const bool x_vec4 = xsz == 4 && (reinterpret_cast<uintptr_t>(xyz) % 16) == 0 && xs % 16 == 0;
    const int t_al = ((reinterpret_cast<uintptr_t>(t) % tsz) == 0 && ts % tsz == 0) ? 1 : 0;
    const int nb = Blocks(m);
    if (xsz == 8) {
        auto k = x_nat ? k_key<double, kLoadNatural> : k_key<double, kLoadBytes>;
        k<<<nb, kThreads, 0, s>>>(xyz, xs, t, ts, t_dtype, t_al, m, A, d_w_.data(), d_pv_.data(), d_cnt_.data());
    } else {
        auto k = x_vec4 ? k_key<float, kLoadVec4> : x_nat ? k_key<float, kLoadNatural> : k_key<float, kLoadBytes>;
        k<<<nb, kThreads, 0, s>>>(xyz, xs, t, ts, t_dtype, t_al, m, A, d_w_.data(), d_pv_.data(), d_cnt_.data());
    }
    CT_CUDA_CHECK(cudaGetLastError());
    k_first_flags<<<Blocks(lcap), kThreads, 0, s>>>(d_ltab_.data(), lcap, d_flag_.data());
    CT_CUDA_CHECK(cudaGetLastError());
    Scan(d_flag_.data(), d_scan0_.data(), m, 1);
    k_resolve<<<nb, kThreads, 0, s>>>(d_ltab_.data(), d_scan0_.data(), m, (uint32_t) cap_v_, d_pv_.data());
    CT_CUDA_CHECK(cudaGetLastError());
    RankArgs R{d_vcount_.data(), d_vlo_.data(), d_vcand_.data(), d_nlo_.data(), d_ncand_.data(), (uint32_t) cap_v_, kp_};
    const int rounds = (int) std::min<uint64_t>((uint64_t) kp_, m);
    for (int r = 0; r < rounds; ++r) {
        k_cand<<<nb, kThreads, 0, s>>>(d_pv_.data(), m, R, r);
        k_take<<<nb, kThreads, 0, s>>>(d_pv_.data(), m, R, r, d_slot_.data(), d_keep_.data());
    }
    CT_CUDA_CHECK(cudaGetLastError());
    Scan(d_keep_.data(), d_scan1_.data(), m, 2);
    CT_CUDA_CHECK(cudaMemcpyAsync(h_cnt_.data(), d_cnt_.data(), sizeof(unsigned long long) * 4, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    st.rejected = h_cnt_.data()[0];
    st.new_voxels = h_cnt_.data()[1];
    st.kept = h_cnt_.data()[2];
    k_reset_lo<<<nb, kThreads, 0, s>>>(d_pv_.data(), m, (uint32_t) cap_v_, d_vlo_.data());
    CT_CUDA_CHECK(cudaGetLastError());
    if (num_voxels_ + st.new_voxels > cap_v_ || num_points_ + st.kept > cap_p_) {
        CT_CUDA_CHECK(cudaStreamSynchronize(s));
        throw CapacityError("world cloud: the points would exceed the capacity (" + std::to_string(num_voxels_) + " + " +
                            std::to_string(st.new_voxels) + " voxels of " + std::to_string(cap_v_) + ", " +
                            std::to_string(num_points_) + " + " + std::to_string(st.kept) + " points of " +
                            std::to_string(cap_p_) + ")");
    }
    k_commit_voxels<<<Blocks(lcap), kThreads, 0, s>>>(d_ltab_.data(), lcap, d_scan0_.data(), num_voxels_, d_table_.data(),
                                                      table_mask_);
    k_commit<<<nb, kThreads, 0, s>>>(d_pv_.data(), d_slot_.data(), d_scan1_.data(), d_w_.data(), m, (uint32_t) cap_v_,
                                     num_voxels_, num_points_, num_submitted_, kp_, d_vcount_.data(), d_vpts_.data(),
                                     d_pxyzt_.data(), d_psrc_.data());
    CT_CUDA_CHECK(cudaGetLastError());
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    num_voxels_ += st.new_voxels;
    num_points_ += st.kept;
    num_submitted_ += m;
    if (stats) *stats = st;
}

void WorldCloud::Add(ContinuousTrajectory *traj, const cticp_cloud_view &c, const uint64_t *segment_ends,
                     const uint32_t *segment_frame_ids, size_t num_segments, cticp_world_cloud_stats *stats) {
    const uint64_t n = c.num_points;
    if (n && !c.data) throw std::invalid_argument("cloud: null data");
    CheckRecordDtypes(c.xyz_dtype, c.t_dtype, traj != nullptr);
    const uint64_t xw = (uint64_t) c.xyz_offset + 3 * (c.xyz_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8);
    const uint64_t tw = c.t_dtype ? (uint64_t) c.t_offset + scan_pack::dtype_size(c.t_dtype) : 0;
    if (xw > c.point_step || tw > c.point_step)
        throw std::invalid_argument("cloud view: a field lies outside the record (point_step)");
    if (traj && traj->Device() != device_) throw std::invalid_argument("the trajectory lives on another device");
    if (!traj && num_segments) throw std::invalid_argument("segments need a trajectory");
    if (traj) traj->CheckSegments(segment_ends, segment_frame_ids, num_segments, n);
    if (n > kMaxCallPoints) throw std::invalid_argument("more than 2^30 points in one call");
    CT_CUDA_CHECK(cudaSetDevice(device_));
    cudaStream_t s = stream_.get();
    if (n == 0) return Ingest(nullptr, 0, c.xyz_dtype, nullptr, 0, 0, 0, stats);
    const uint64_t bytes = SpanBytes(n, c.point_step, std::max(xw, tw), "cloud");
    d_rec_.reserve(bytes, s);
    CT_CUDA_CHECK(cudaMemcpyAsync(d_rec_.data(), c.data, bytes, cudaMemcpyHostToDevice, s));
    if (!traj) {
        Ingest(d_rec_.data() + c.xyz_offset, c.point_step, c.xyz_dtype, d_rec_.data() + c.t_offset, c.point_step, c.t_dtype,
               n, stats);
        return;
    }
    cticp_device_scan scan{};
    scan.xyz = d_rec_.data() + c.xyz_offset;
    scan.xyz_stride_bytes = c.point_step;
    scan.t = d_rec_.data() + c.t_offset;
    scan.t_stride_bytes = c.point_step;
    scan.num_points = n;
    scan.xyz_dtype = c.xyz_dtype;
    scan.t_dtype = c.t_dtype;
    AddDevice(traj, scan, segment_ends, segment_frame_ids, num_segments, stats, s);
}

void WorldCloud::AddDevice(ContinuousTrajectory *traj, const cticp_device_scan &scan, const uint64_t *segment_ends,
                           const uint32_t *segment_frame_ids, size_t num_segments, cticp_world_cloud_stats *stats,
                           cudaStream_t stream) {
    const uint64_t n = scan.num_points;
    CheckRecordDtypes(scan.xyz_dtype, scan.t_dtype, traj != nullptr);
    if (n && (!scan.xyz || (scan.t_dtype && !scan.t))) throw std::invalid_argument("scan: null xyz / t");
    if (traj && traj->Device() != device_) throw std::invalid_argument("the trajectory lives on another device");
    if (!traj && num_segments) throw std::invalid_argument("segments need a trajectory");
    if (traj) traj->CheckSegments(segment_ends, segment_frame_ids, num_segments, n);
    if (n > kMaxCallPoints) throw std::invalid_argument("more than 2^30 points in one call");
    CT_CUDA_CHECK(cudaSetDevice(device_));
    if (n == 0) return Ingest(nullptr, 0, scan.xyz_dtype, nullptr, 0, 0, 0, stats);
    const uint64_t xsz = scan.xyz_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8;
    RequireDeviceRange(scan.xyz, SpanBytes(n, scan.xyz_stride_bytes, 3 * xsz, "xyz"), device_, "xyz");
    if (scan.t_dtype)
        RequireDeviceRange(scan.t, SpanBytes(n, scan.t_stride_bytes, scan_pack::dtype_size(scan.t_dtype), "t"), device_, "t");
    cudaStream_t s = stream_.get();
    if (stream != s) {   // behind the caller's work on its records
        CT_CUDA_CHECK(cudaEventRecord(ev_in_.get(), stream));
        CT_CUDA_CHECK(cudaStreamWaitEvent(s, ev_in_.get(), 0));
    }
    if (!traj) {
        Ingest(static_cast<const unsigned char *>(scan.xyz), scan.xyz_stride_bytes, scan.xyz_dtype,
               static_cast<const unsigned char *>(scan.t), scan.t_stride_bytes, scan.t_dtype, n, stats);
        return;
    }
    // the world points are the trajectory's own transform (cticp_trajectory_transform_device), bit for bit
    d_w_.reserve(n, s);
    traj->TransformDevice(scan, segment_ends, segment_frame_ids, num_segments, WorldSink(d_w_.data(), n), s);
    const unsigned char *w = reinterpret_cast<const unsigned char *>(d_w_.data());
    Ingest(w, sizeof(double4), CTICP_DTYPE_FLOAT64, w + 24, sizeof(double4), CTICP_DTYPE_FLOAT64, n, stats);
}

void WorldCloud::AddOdometry(Engine &engine, cticp_world_cloud_stats *stats) {
    if (engine.Device() != device_) throw std::invalid_argument("the odometry lives on another device");
    CT_CUDA_CHECK(cudaSetDevice(device_));
    cudaStream_t s = stream_.get();
    const cticp_cloud_sink probe{};
    const uint64_t n = (uint64_t) engine.WritePointsDevice(CTICP_POINTS_ALL_CORRECTED, probe, s);
    if (n > kMaxCallPoints) throw std::invalid_argument("more than 2^30 points in one call");
    if (n == 0) return Ingest(nullptr, 0, CTICP_DTYPE_FLOAT64, nullptr, 0, 0, 0, stats);
    d_w_.reserve(n, s);
    // the points cticp_odometry_write_points_device(CTICP_POINTS_ALL_CORRECTED) writes, ordered before this stream
    engine.WritePointsDevice(CTICP_POINTS_ALL_CORRECTED, WorldSink(d_w_.data(), n), s);
    const unsigned char *w = reinterpret_cast<const unsigned char *>(d_w_.data());
    Ingest(w, sizeof(double4), CTICP_DTYPE_FLOAT64, w + 24, sizeof(double4), CTICP_DTYPE_FLOAT64, n, stats);
}

void WorldCloud::EnqueueExport(unsigned char *sink_data, const cticp_cloud_sink &sink, uint64_t *d_src, uint64_t m) {
    cudaStream_t s = stream_.get();
    if (num_voxels_ == 0 || m == 0) return;
    Scan(d_vcount_.data(), d_off_.data(), num_voxels_, 3);
    SinkArgs sa{};
    if (sink_data) {
        const size_t osz = sink.xyz_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8, otsz = sink.t_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8;
        sa.data = sink_data;
        sa.step = sink.point_step;
        sa.xoff = sink.xyz_offset;
        sa.toff = sink.t_offset;
        sa.xdt = sink.xyz_dtype;
        sa.tdt = sink.t_dtype;
        sa.x_aligned = ((reinterpret_cast<uintptr_t>(sink_data) + sink.xyz_offset) % osz == 0 && sink.point_step % osz == 0) ? 1 : 0;
        sa.t_aligned = ((reinterpret_cast<uintptr_t>(sink_data) + sink.t_offset) % otsz == 0 && sink.point_step % otsz == 0) ? 1 : 0;
    }
    k_export<<<Blocks(num_voxels_), kThreads, 0, s>>>(d_vcount_.data(), d_off_.data(), d_vpts_.data(), d_pxyzt_.data(),
                                                      d_psrc_.data(), num_voxels_, kp_, m, sa, d_src);
    CT_CUDA_CHECK(cudaGetLastError());
}

int64_t WorldCloud::Export(const cticp_cloud_sink &sink, uint64_t *src_index) {
    const uint64_t n = NumPoints();
    if (!sink.world) throw std::invalid_argument("sink: world must be set (a world cloud holds world coordinates)");
    const uint64_t m = std::min<uint64_t>(sink.capacity_points, n);
    if (m == 0 || (!sink.data && !src_index)) return (int64_t) n;
    if (sink.data) CheckSink(sink);
    CT_CUDA_CHECK(cudaSetDevice(device_));
    cudaStream_t s = stream_.get();
    uint64_t out_bytes = 0;
    if (sink.data) {
        out_bytes = SpanBytes(m, sink.point_step, SinkRecordWidth(sink), "sink");
        d_sink_.reserve(out_bytes, s);
        // the sink goes over as it is: its bytes outside x, y, z and t stay the caller's
        CT_CUDA_CHECK(cudaMemcpyAsync(d_sink_.data(), sink.data, out_bytes, cudaMemcpyHostToDevice, s));
    }
    if (src_index) d_src_out_.reserve(m, s);
    EnqueueExport(sink.data ? d_sink_.data() : nullptr, sink, src_index ? d_src_out_.data() : nullptr, m);
    if (sink.data) CT_CUDA_CHECK(cudaMemcpyAsync(sink.data, d_sink_.data(), out_bytes, cudaMemcpyDeviceToHost, s));
    if (src_index)
        CT_CUDA_CHECK(cudaMemcpyAsync(src_index, d_src_out_.data(), sizeof(uint64_t) * m, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    return (int64_t) n;
}

int64_t WorldCloud::ExportDevice(const cticp_cloud_sink &sink, uint64_t *src_index, cudaStream_t stream) {
    const uint64_t n = NumPoints();
    if (!sink.world) throw std::invalid_argument("sink: world must be set (a world cloud holds world coordinates)");
    const uint64_t m = std::min<uint64_t>(sink.capacity_points, n);
    if (m == 0 || (!sink.data && !src_index)) return (int64_t) n;
    if (sink.data) CheckSink(sink);
    CT_CUDA_CHECK(cudaSetDevice(device_));
    if (sink.data)
        RequireDeviceRange(sink.data, SpanBytes(m, sink.point_step, SinkRecordWidth(sink), "sink"), device_, "sink");
    if (src_index) RequireDeviceRange(src_index, sizeof(uint64_t) * m, device_, "src_index");
    cudaStream_t s = stream_.get();
    // ordered both ways with the caller's stream: behind what it queued before (the sink's allocation), ahead of what it
    // queues next
    CT_CUDA_CHECK(cudaEventRecord(ev_in_.get(), stream));
    CT_CUDA_CHECK(cudaStreamWaitEvent(s, ev_in_.get(), 0));
    EnqueueExport(static_cast<unsigned char *>(sink.data), sink, src_index, m);
    CT_CUDA_CHECK(cudaEventRecord(ev_out_.get(), s));
    CT_CUDA_CHECK(cudaStreamWaitEvent(stream, ev_out_.get(), 0));
    return (int64_t) n;
}

}  // namespace cticp
