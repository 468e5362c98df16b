// dataset.cu — dataset sequences on the device: the NCLT packet index and hit decode, the KITTI frame filter and the
// per-frame timestamp ranges; and the host readers of PLY headers and ground-truth files.
//
// This file is compiled with -fmad=false: the decode is the reference's fp64 multiply then subtract, and the filter's
// axis, normalisation, rotation matrix and product are Eigen's fp64 operations, operation for operation.
// The NCLT index runs in three steps on the handle's stream:
//   1. one thread per 8-byte word marks the words equal to the magic (0xAD9CAD9CAD9CAD9C) whose 24-byte header fits;
//      tiles of kThreads words, taken from an atomic ticket, compact them in order with tile_lookback.cuh;
//   2. one thread per candidate checks that its successor c + 24 + 8 num_hits is the next candidate (the first must be at
//      0, and what follows the last must be the end or a partial packet), and records the packet;
//   3. only when a link fails (a hit whose 8 bytes equal the magic: laser id 173), one thread walks the packets from
//      offset 0, as the reference reads them, and that walk is the index.
// The host then receives each packet's hit count and utime (12 bytes per packet), forms the frames, and uploads the
// packets' first hits; a read decodes one thread per hit, finding its packet by binary search.
#include "dataset.h"

#include <algorithm>
#include <cerrno>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>

#include "device_checks.h"
#include "device_map.h"
#include "engine.h"
#include "record_io.cuh"
#include "scan_pack.cuh"
#include "se3.cuh"
#include "tile_lookback.cuh"

namespace cticp {

namespace {

constexpr int kThreads = 256;
constexpr unsigned long long kMagic = 0xAD9CAD9CAD9CAD9Cull;   // 4 x u16 44444, little endian
constexpr uint64_t kHeader = 24;
// walk / chain results: status and byte offset
enum { kEnd = 0, kTruncated = 1, kBadMagic = 2 };

int Blocks(uint64_t n, int sms) {
    return (int) std::max<uint64_t>(1, std::min<uint64_t>((n + kThreads - 1) / kThreads, (uint64_t) sms * 8));
}

__device__ __forceinline__ uint32_t load_u32(const unsigned long long *w, uint64_t byte) {   // 4-aligned
    return reinterpret_cast<const uint32_t *>(w)[byte >> 2];
}
__device__ __forceinline__ uint64_t load_utime(const unsigned long long *w, uint64_t pkt) {   // byte pkt + 12
    return (uint64_t) load_u32(w, pkt + 12) | ((uint64_t) load_u32(w, pkt + 16) << 32);
}

// desc[tiles] is the ticket; cand receives the byte offsets of the marked words in order; *count the total
__global__ void k_candidates(const unsigned long long *__restrict__ words, uint64_t n_words, uint64_t n_bytes,
                             uint64_t tiles, unsigned long long *desc, uint64_t *cand, uint64_t cap,
                             unsigned long long *count) {
    __shared__ uint32_t s_warp[kThreads / 32];
    __shared__ uint32_t s_tile, s_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (;;) {
        if (threadIdx.x == 0) s_tile = (uint32_t) atomicAdd(&desc[tiles], 1ull);
        __syncthreads();
        const uint64_t tile = s_tile;
        if (tile >= tiles) return;
        const uint64_t w = tile * kThreads + threadIdx.x;
        const bool hit = w < n_words && w * 8 + kHeader <= n_bytes && __ldg(&words[w]) == kMagic;
        const unsigned ballot = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) s_warp[warp] = __popc(ballot);
        __syncthreads();
        uint32_t before = __popc(ballot & ((1u << lane) - 1)), total = 0;
        for (int k = 0; k < kThreads / 32; ++k) {
            const uint32_t v = s_warp[k];
            if (k < warp) before += v;
            total += v;
        }
        if (warp == 0) {
            const uint32_t base = tile_lookback(desc, (int) tile, total);
            if (lane == 0) s_base = base;
        }
        __syncthreads();
        if (hit && (uint64_t) s_base + before < cap) cand[(uint64_t) s_base + before] = w * 8;
        if (threadIdx.x == 0 && tile == tiles - 1) *count = (unsigned long long) s_base + total;
        __syncthreads();
    }
}

// result[0] |= 1 when the chain breaks; result[1..2]: the status and offset of what follows the last complete packet;
// result[3] = 1 when the last candidate's packet is partial
__global__ void k_chain(const unsigned long long *__restrict__ words, uint64_t n_bytes, const uint64_t *cand, uint64_t k_n,
                        uint32_t *nh, uint64_t *ut, unsigned long long *result) {
    for (uint64_t k = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; k < k_n; k += (uint64_t) gridDim.x * blockDim.x) {
        const uint64_t c = cand[k];
        const uint32_t n = load_u32(words, c + 8);
        nh[k] = n;
        ut[k] = load_utime(words, c);
        const uint64_t succ = c + kHeader + 8ull * n;
        bool ok = k > 0 || c == 0;
        if (k + 1 < k_n) {
            ok = ok && succ == cand[k + 1];
        } else if (succ > n_bytes) {   // the last packet is partial
            result[1] = kTruncated;
            result[2] = c;
            result[3] = 1;
        } else if (succ == n_bytes) {
            result[1] = kEnd;
            result[2] = succ;
        } else {   // a tail of fewer than 24 bytes that starts with the magic or is shorter than it, else a bad header
            const uint64_t tail = n_bytes - succ;
            ok = ok && tail < kHeader && (tail < 8 || __ldg(&words[succ >> 3]) == kMagic);
            result[1] = kTruncated;
            result[2] = succ;
        }
        if (!ok) atomicOr(&result[0], 1ull);
    }
}

// the reference's sequential read (NCLTIterator::NextBatch), one thread: result[1..3] = status, offset, packets
__global__ void k_walk(const unsigned long long *__restrict__ words, uint64_t n_bytes, uint64_t *off_out, uint32_t *nh,
                       uint64_t *ut, unsigned long long *result) {
    uint64_t off = 0, p = 0;
    int status = kEnd;
    while (off < n_bytes) {
        if (n_bytes - off >= 8 && words[off >> 3] != kMagic) {
            status = kBadMagic;
            break;
        }
        if (n_bytes - off < kHeader) {
            status = kTruncated;
            break;
        }
        const uint32_t n = load_u32(words, off + 8);
        const uint64_t end = off + kHeader + 8ull * n;
        if (end > n_bytes) {
            status = kTruncated;
            break;
        }
        off_out[p] = off;
        nh[p] = n;
        ut[p] = load_utime(words, off);
        ++p;
        off = end;
    }
    result[1] = (unsigned long long) status;
    result[2] = off;
    result[3] = p;
}

// hits [hit0, hit0 + total) of packets [p0, p1): x = (double) u * 0.005 - 100.0, t = (double) utime
__global__ void k_decode(const unsigned long long *__restrict__ words, const uint64_t *__restrict__ pkt_off,
                         const uint64_t *__restrict__ hit_start, uint64_t p0, uint64_t p1, uint64_t hit0,
                         uint64_t total, GenSink sink) {
    for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < total && i < sink.cap;
         i += (uint64_t) gridDim.x * blockDim.x) {
        const uint64_t h = hit0 + i;
        uint64_t lo = p0, hi = p1;   // the last packet whose first hit is <= h
        while (hi - lo > 1) {
            const uint64_t mid = lo + (hi - lo) / 2;
            if (__ldg(&hit_start[mid]) <= h) lo = mid;
            else hi = mid;
        }
        const uint64_t pkt = __ldg(&pkt_off[lo]);
        const unsigned long long rec = __ldg(&words[(pkt + kHeader) / 8 + (h - __ldg(&hit_start[lo]))]);
        const double t = __ull2double_rn(load_utime(words, pkt));
        V3 p;
        p.x = __dsub_rn(__dmul_rn((double) (uint32_t) (rec & 0xFFFFu), 0.005), 100.0);
        p.y = __dsub_rn(__dmul_rn((double) (uint32_t) ((rec >> 16) & 0xFFFFu), 0.005), 100.0);
        p.z = __dsub_rn(__dmul_rn((double) (uint32_t) ((rec >> 32) & 0xFFFFu), 0.005), 100.0);
        store_gen_record(sink, i, p, t);
    }
}

__global__ void k_frame_ends(const uint64_t *frame_start, uint64_t first, uint64_t m, uint64_t *ends) {
    for (uint64_t k = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; k < m; k += (uint64_t) gridDim.x * blockDim.x)
        ends[k] = frame_start[first + k + 1] - frame_start[first];
}

struct ScanArgs {
    const unsigned char *xyz, *t;
    uint64_t xs, ts, n;
    int xdt, tdt, t_aligned;
};

template <typename XT>
__device__ __forceinline__ V3 load_point(const ScanArgs &a, uint64_t i, bool aligned) {
    XT x, y, z;
    if (aligned) {   // plain loads, not __ldg: the filter may write these records in place
        const XT *q = reinterpret_cast<const XT *>(a.xyz + i * a.xs);
        x = q[0]; y = q[1]; z = q[2];
    } else {
        load_xyz<XT, kLoadBytes>(a.xyz + i * a.xs, x, y, z);
    }
    return V3{(double) x, (double) y, (double) z};
}

// kitti_frame_filter, dataset.cpp:85-110; sin_a / cos_a of 0.205 * M_PI / 180.0 from the host C library
__global__ void k_kitti_filter(ScanArgs a, int x_aligned, double sin_a, double cos_a, GenSink sink) {
    for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < a.n; i += (uint64_t) gridDim.x * blockDim.x) {
        const V3 p = a.xdt == CTICP_DTYPE_FLOAT32 ? load_point<float>(a, i, x_aligned) : load_point<double>(a, i, x_aligned);
        const double t = sink.tdt ? load_timestamp(a.t + i * a.ts, a.tdt, a.t_aligned) : 0.0;
        V3 q{0.0, 0.0, 0.0};
        if (p.z > -5.0) {
            const double ux = 0.0, uy = 0.0, uz = 1.0;   // Eigen cross(old_pt, uz)
            double ax = p.y * uz - p.z * uy, ay = p.z * ux - p.x * uz, az = p.x * uy - p.y * ux;
            const double sq = (ax * ax + ay * ay) + az * az;   // normalize(): v / sqrt(squaredNorm) when > 0
            if (sq > 0.0) {
                const double s = sqrt(sq);
                ax = ax / s;
                ay = ay / s;
                az = az / s;
            }
            // AngleAxis::toRotationMatrix
            const double sx = sin_a * ax, sy = sin_a * ay, sz = sin_a * az;
            const double cx = (1.0 - cos_a) * ax, cy = (1.0 - cos_a) * ay, cz = (1.0 - cos_a) * az;
            double tmp = cx * ay;
            const double r01 = tmp - sz, r10 = tmp + sz;
            tmp = cx * az;
            const double r02 = tmp + sy, r20 = tmp - sy;
            tmp = cy * az;
            const double r12 = tmp - sx, r21 = tmp + sx;
            const double r00 = cx * ax + cos_a, r11 = cy * ay + cos_a, r22 = cz * az + cos_a;
            q.x = (r00 * p.x + r01 * p.y) + r02 * p.z;
            q.y = (r10 * p.x + r11 * p.y) + r12 * p.z;
            q.z = (r20 * p.x + r21 * p.y) + r22 * p.z;
        }
        store_gen_record(sink, i, q, t);
    }
}

// one CTA per frame: (min, max) of its timestamps, NaN for both when one is NaN, (+inf, -inf) when it is empty
__global__ void k_time_ranges(ScanArgs a, const uint64_t *ends, uint64_t m, double *out) {
    __shared__ double s_mn[kThreads / 32], s_mx[kThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint64_t f = blockIdx.x; f < m; f += gridDim.x) {
        const uint64_t b = f ? ends[f - 1] : 0, e = ends[f];
        double mn = INFINITY, mx = -INFINITY;
        bool nan = false;
        for (uint64_t i = b + threadIdx.x; i < e && i < a.n; i += blockDim.x) {
            const double v = load_timestamp(a.t + i * a.ts, a.tdt, a.t_aligned);
            nan |= v != v;
            mn = fmin(mn, v);
            mx = fmax(mx, v);
        }
        for (int o = 16; o; o >>= 1) {
            mn = fmin(mn, __shfl_xor_sync(0xffffffffu, mn, o));
            mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        }
        if (lane == 0) {
            s_mn[warp] = mn;
            s_mx[warp] = mx;
        }
        nan = __syncthreads_or(nan);
        if (threadIdx.x == 0) {
            for (int k = 1; k < kThreads / 32; ++k) {
                mn = fmin(mn, s_mn[k]);
                mx = fmax(mx, s_mx[k]);
            }
            out[2 * f] = nan ? NAN : mn;
            out[2 * f + 1] = nan ? NAN : mx;
        }
        __syncthreads();
    }
}

void RequireAligned(const void *p, uint64_t align, const char *what) {
    if (reinterpret_cast<uintptr_t>(p) % align)
        throw std::invalid_argument(std::string(what) + " is not " + std::to_string(align) + "-byte aligned");
}

int SmCount(int device) {
    int sms = 1;
    CT_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    return sms;
}

// the scan's dtypes and its buffers inside device allocations of `device`; x, y, z only when `need_xyz`, the timestamp
// only when `need_t`
ScanArgs CheckDeviceScan(const cticp_device_scan &scan, int device, bool need_t, bool need_xyz = true) {
    const uint64_t n = scan.num_points;
    if (need_xyz && scan.xyz_dtype != CTICP_DTYPE_FLOAT32 && scan.xyz_dtype != CTICP_DTYPE_FLOAT64)
        throw std::invalid_argument("scan: x/y/z must be FLOAT32 or FLOAT64");
    if (need_t && scan_pack::dtype_size(scan.t_dtype) == 0) throw std::invalid_argument("scan: unknown timestamp dtype");
    const uint64_t xsz = scan.xyz_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8;
    if (n && need_xyz && !scan.xyz) throw std::invalid_argument("scan: null xyz");
    if (n && need_t && !scan.t) throw std::invalid_argument("scan: null t");
    if (n && need_xyz) RequireDeviceRange(scan.xyz, SpanBytes(n, scan.xyz_stride_bytes, 3 * xsz, "xyz"), device, "xyz");
    if (n && need_t)
        RequireDeviceRange(scan.t, SpanBytes(n, scan.t_stride_bytes, scan_pack::dtype_size(scan.t_dtype), "t"), device, "t");
    ScanArgs a{};
    a.xyz = static_cast<const unsigned char *>(scan.xyz);
    a.t = static_cast<const unsigned char *>(scan.t);
    a.xs = scan.xyz_stride_bytes;
    a.ts = scan.t_stride_bytes;
    a.n = n;
    a.xdt = scan.xyz_dtype;
    a.tdt = need_t ? scan.t_dtype : 0;
    const unsigned tsz = scan_pack::dtype_size(scan.t_dtype);
    a.t_aligned = need_t && tsz && reinterpret_cast<uintptr_t>(scan.t) % tsz == 0 && scan.t_stride_bytes % tsz == 0;
    return a;
}

int XyzAligned(const cticp_device_scan &scan) {
    const uint64_t xsz = scan.xyz_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8;
    return reinterpret_cast<uintptr_t>(scan.xyz) % xsz == 0 && scan.xyz_stride_bytes % xsz == 0;
}

void CheckFilterSink(const cticp_cloud_sink &sink, uint64_t n) {
    CheckSink(sink);
    if (sink.world) throw std::invalid_argument("sink: world must be 0 (the filter writes sensor coordinates)");
    if (n && (!sink.data || sink.capacity_points < n))
        throw std::invalid_argument("sink: room for every point of the scan is required");
}

void LaunchFilter(int device, const cticp_device_scan &scan, const ScanArgs &a, const cticp_cloud_sink &sink,
                  unsigned char *out, cudaStream_t s) {
    // the angle as the reference writes it: KITTI_GLOBAL_VERTICAL_ANGLE_OFFSET * M_PI / 180.0
    const double angle = 0.205 * M_PI / 180.0;
    k_kitti_filter<<<Blocks(a.n, SmCount(device)), kThreads, 0, s>>>(a, XyzAligned(scan), std::sin(angle),
                                                                     std::cos(angle), MakeGenSink(out, sink, a.n));
    CT_CUDA_CHECK(cudaGetLastError());
}

// a cticp_device_scan over host records copied to `base` on the device
cticp_device_scan DeviceScanOfCloud(const cticp_cloud_view &c, const unsigned char *base) {
    cticp_device_scan s{};
    s.xyz = base + c.xyz_offset;
    s.xyz_stride_bytes = c.point_step;
    s.t = base + c.t_offset;
    s.t_stride_bytes = c.point_step;
    s.num_points = c.num_points;
    s.xyz_dtype = c.xyz_dtype;
    s.t_dtype = c.t_dtype;
    return s;
}

uint64_t CloudBytes(const cticp_cloud_view &c, bool with_t) {
    if (!c.data) throw std::invalid_argument("cloud: null data");
    if (c.xyz_dtype != CTICP_DTYPE_FLOAT32 && c.xyz_dtype != CTICP_DTYPE_FLOAT64)
        throw std::invalid_argument("cloud: x/y/z must be FLOAT32 or FLOAT64");
    uint64_t width = (uint64_t) c.xyz_offset + 3 * (c.xyz_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8);
    if (with_t) {
        if (scan_pack::dtype_size(c.t_dtype) == 0) throw std::invalid_argument("cloud: unknown timestamp dtype");
        width = std::max<uint64_t>(width, (uint64_t) c.t_offset + scan_pack::dtype_size(c.t_dtype));
    }
    if (width > c.point_step) throw std::invalid_argument("cloud: a field lies outside the record (point_step)");
    return SpanBytes(c.num_points, c.point_step, width, "cloud");
}

}  // namespace

// ---- NCLT ------------------------------------------------------------------------------------------------------------
NcltHits::NcltHits(const void *bytes, uint64_t n_bytes, uint32_t num_aggregated, bool final, int device, bool on_device,
                   cudaStream_t stream)
    : device_(device) {
    if (num_aggregated == 0) throw std::invalid_argument("num_aggregated must be >= 1");
    if (n_bytes && !bytes) throw std::invalid_argument("null bytes");
    // the look-back of the index carries 32-bit counts: at most 2^32 - 1 words, so the candidates fit
    if (n_bytes / 8 >= 0xFFFFFFFFull) throw std::invalid_argument("more than 32 GiB of bytes in one handle");
    CT_CUDA_CHECK(cudaSetDevice(device_));
    if (on_device && n_bytes) RequireDeviceRange(bytes, n_bytes, device_, "bytes");
    sms_ = SmCount(device_);
    stream_ = cticp::Stream(cudaStreamNonBlocking);
    ev_in_ = Event(cudaEventDisableTiming);
    ev_out_ = Event(cudaEventDisableTiming);
    cudaStream_t s = stream_.get();
    const uint64_t n_words = (n_bytes + 7) / 8;
    d_bytes_.reserve(std::max<uint64_t>(n_words, 1), s);
    if (n_words) CT_CUDA_CHECK(cudaMemsetAsync(d_bytes_.data() + n_words - 1, 0, 8, s));
    if (on_device) {
        CT_CUDA_CHECK(cudaEventRecord(ev_in_.get(), stream));
        CT_CUDA_CHECK(cudaStreamWaitEvent(s, ev_in_.get(), 0));
    }
    if (n_bytes)
        CT_CUDA_CHECK(cudaMemcpyAsync(d_bytes_.data(), bytes, n_bytes,
                                      on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s));
    Index(n_bytes, num_aggregated, final);
}

NcltHits::~NcltHits() {
    if (stream_.get()) {
        cudaSetDevice(device_);
        cudaStreamSynchronize(stream_.get());
    }
}

void NcltHits::Index(uint64_t n_bytes, uint32_t num_aggregated, bool final) {
    cudaStream_t s = stream_.get();
    const uint64_t n_words = (n_bytes + 7) / 8, tiles = std::max<uint64_t>((n_words + kThreads - 1) / kThreads, 1);
    const uint64_t max_pkts = n_bytes / kHeader + 1;
    DeviceArray<unsigned long long> desc, result;   // result: [0] chain broken, [1] status, [2] offset, [3] packets, [4] K
    DeviceArray<uint64_t> cand, ut;
    DeviceArray<uint32_t> nh;
    desc.reserve(tiles + 1, s);
    result.reserve(5, s);
    cand.reserve(max_pkts, s);
    ut.reserve(max_pkts, s);
    nh.reserve(max_pkts, s);
    CT_CUDA_CHECK(cudaMemsetAsync(desc.data(), 0, sizeof(unsigned long long) * (tiles + 1), s));
    CT_CUDA_CHECK(cudaMemsetAsync(result.data(), 0, sizeof(unsigned long long) * 5, s));
    int per_sm = 1;
    CT_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_candidates, kThreads, 0));
    k_candidates<<<(int) std::min<uint64_t>(tiles, (uint64_t) sms_ * std::max(per_sm, 1)), kThreads, 0, s>>>(
        d_bytes_.data(), n_words, n_bytes, tiles, desc.data(), cand.data(), max_pkts, result.data() + 4);
    CT_CUDA_CHECK(cudaGetLastError());
    unsigned long long k_n = 0;
    CT_CUDA_CHECK(cudaMemcpyAsync(&k_n, result.data() + 4, sizeof(k_n), cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    unsigned long long r[4] = {1, 0, 0, 0};   // more candidates than packets fit: not a chain
    if (k_n && k_n <= max_pkts) {
        k_chain<<<Blocks(k_n, sms_), kThreads, 0, s>>>(d_bytes_.data(), n_bytes, cand.data(), k_n, nh.data(), ut.data(),
                                                       result.data());
        CT_CUDA_CHECK(cudaGetLastError());
        CT_CUDA_CHECK(cudaMemcpyAsync(r, result.data(), sizeof(r), cudaMemcpyDeviceToHost, s));
        CT_CUDA_CHECK(cudaStreamSynchronize(s));
    }
    uint64_t packets;
    if (r[0] == 0) {
        packets = k_n - r[3];
    } else {   // the fallback: the reference's sequential read
        walked_ = true;
        CT_CUDA_CHECK(cudaMemsetAsync(result.data(), 0, sizeof(unsigned long long) * 4, s));
        k_walk<<<1, 1, 0, s>>>(d_bytes_.data(), n_bytes, cand.data(), nh.data(), ut.data(), result.data());
        CT_CUDA_CHECK(cudaGetLastError());
        CT_CUDA_CHECK(cudaMemcpyAsync(r, result.data(), sizeof(r), cudaMemcpyDeviceToHost, s));
        CT_CUDA_CHECK(cudaStreamSynchronize(s));
        packets = r[3];
        if (r[1] == kBadMagic)
            throw std::invalid_argument("NCLT: the packet header at byte offset " + std::to_string(r[2]) +
                                        " does not have a matching magic number");
    }
    if (final && r[1] == kTruncated)
        throw std::invalid_argument("NCLT: truncated packet at byte offset " + std::to_string(r[2]));
    std::vector<uint64_t> off(packets), utime(packets);
    std::vector<uint32_t> hits(packets);
    if (packets) {
        CT_CUDA_CHECK(cudaMemcpyAsync(off.data(), cand.data(), sizeof(uint64_t) * packets, cudaMemcpyDeviceToHost, s));
        CT_CUDA_CHECK(cudaMemcpyAsync(utime.data(), ut.data(), sizeof(uint64_t) * packets, cudaMemcpyDeviceToHost, s));
        CT_CUDA_CHECK(cudaMemcpyAsync(hits.data(), nh.data(), sizeof(uint32_t) * packets, cudaMemcpyDeviceToHost, s));
        CT_CUDA_CHECK(cudaStreamSynchronize(s));
    }
    const uint64_t A = agg_ = num_aggregated;
    const uint64_t frames = final ? (packets + A - 1) / A : packets / A;
    packets_ = std::min(packets, frames * A);
    bytes_used_ = packets_ ? off[packets_ - 1] + kHeader + 8ull * hits[packets_ - 1] : 0;
    std::vector<uint64_t> hit_start(packets_ + 1, 0);
    frame_start_.assign(frames + 1, 0);
    info_.assign(frames, cticp_nclt_frame{0, NAN, NAN});
    for (uint64_t p = 0; p < packets_; ++p) {
        hit_start[p + 1] = hit_start[p] + hits[p];
        cticp_nclt_frame &fi = info_[p / A];
        if (hits[p] == 0) continue;
        const double t = (double) utime[p];
        if (fi.num_points == 0) fi.t_first = fi.t_max = t;
        fi.t_max = std::max(fi.t_max, t);
        fi.num_points += hits[p];
    }
    for (uint64_t f = 0; f < frames; ++f) frame_start_[f + 1] = frame_start_[f] + info_[f].num_points;
    d_pkt_off_ = std::move(cand);
    d_hit_start_.reserve(packets_ + 1, s);
    d_frame_start_.reserve(frames + 1, s);
    CT_CUDA_CHECK(cudaMemcpyAsync(d_hit_start_.data(), hit_start.data(), sizeof(uint64_t) * (packets_ + 1),
                                  cudaMemcpyHostToDevice, s));
    CT_CUDA_CHECK(cudaMemcpyAsync(d_frame_start_.data(), frame_start_.data(), sizeof(uint64_t) * (frames + 1),
                                  cudaMemcpyHostToDevice, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
}

void NcltHits::FrameInfo(uint64_t first, uint64_t m, cticp_nclt_frame *out) const {
    if (m && !out) throw std::invalid_argument("null out");
    if (first > NumFrames() || m > NumFrames() - first) throw std::invalid_argument("frames outside the handle");
    std::copy(info_.begin() + first, info_.begin() + first + m, out);
}

void NcltHits::CheckRead(uint64_t first, uint64_t m, const cticp_cloud_sink &sink) const {
    if (first > NumFrames() || m > NumFrames() - first) throw std::invalid_argument("frames outside the handle");
    CheckSink(sink);
    if (sink.world) throw std::invalid_argument("sink: world must be 0 (NCLT hits are sensor coordinates)");
}

void NcltHits::LaunchDecode(uint64_t first, uint64_t m, unsigned char *data, const cticp_cloud_sink &sink, uint64_t cap,
                            uint64_t *frame_ends) {
    cudaStream_t s = stream_.get();
    const uint64_t hit0 = frame_start_[first], total = frame_start_[first + m] - hit0;
    if (data && cap && total) {
        const uint64_t p0 = first * agg_, p1 = std::min(packets_, (first + m) * agg_);   // the frames' packets
        k_decode<<<Blocks(std::min(total, cap), sms_), kThreads, 0, s>>>(d_bytes_.data(), d_pkt_off_.data(),
                                                                         d_hit_start_.data(), p0, p1, hit0, total,
                                                                         MakeGenSink(data, sink, cap));
        CT_CUDA_CHECK(cudaGetLastError());
    }
    k_frame_ends<<<Blocks(m, sms_), kThreads, 0, s>>>(d_frame_start_.data(), first, m, frame_ends);
    CT_CUDA_CHECK(cudaGetLastError());
}

int64_t NcltHits::ReadFrames(uint64_t first, uint64_t m, const cticp_cloud_sink &sink, uint64_t *frame_ends) {
    CheckRead(first, m, sink);
    if (m && !frame_ends) throw std::invalid_argument("null frame_ends");
    if (m == 0) return 0;
    const uint64_t count = frame_start_[first + m] - frame_start_[first];
    const uint64_t cap = std::min<uint64_t>(sink.data ? sink.capacity_points : 0, count);
    const uint64_t out_bytes = cap ? SpanBytes(cap, sink.point_step, SinkRecordWidth(sink), "sink") : 0;
    CT_CUDA_CHECK(cudaSetDevice(device_));
    cudaStream_t s = stream_.get();
    d_out_.reserve(std::max<uint64_t>(out_bytes, 1), s);
    d_ends_.reserve(m, s);
    // the sink goes over as it is: its bytes outside x, y, z and t stay the caller's
    if (out_bytes) CT_CUDA_CHECK(cudaMemcpyAsync(d_out_.data(), sink.data, out_bytes, cudaMemcpyHostToDevice, s));
    LaunchDecode(first, m, out_bytes ? d_out_.data() : nullptr, sink, cap, d_ends_.data());
    if (out_bytes) CT_CUDA_CHECK(cudaMemcpyAsync(sink.data, d_out_.data(), out_bytes, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaMemcpyAsync(frame_ends, d_ends_.data(), sizeof(uint64_t) * m, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    return (int64_t) count;
}

void NcltHits::ReadFramesDevice(uint64_t first, uint64_t m, const cticp_cloud_sink &sink, uint64_t *frame_ends,
                                cudaStream_t stream) {
    CheckRead(first, m, sink);
    if (m && !frame_ends) throw std::invalid_argument("null frame_ends");
    if (m == 0) return;
    const uint64_t count = frame_start_[first + m] - frame_start_[first];
    const uint64_t cap = std::min<uint64_t>(sink.data ? sink.capacity_points : 0, count);
    CT_CUDA_CHECK(cudaSetDevice(device_));
    RequireAligned(frame_ends, 8, "frame_ends");
    RequireDeviceRange(frame_ends, sizeof(uint64_t) * m, device_, "frame_ends");
    if (cap) RequireDeviceRange(sink.data, SpanBytes(cap, sink.point_step, SinkRecordWidth(sink), "sink"), device_, "sink");
    cudaStream_t s = stream_.get();
    // ordered both ways with the caller's stream: behind what it queued before, ahead of what it queues next
    CT_CUDA_CHECK(cudaEventRecord(ev_in_.get(), stream));
    CT_CUDA_CHECK(cudaStreamWaitEvent(s, ev_in_.get(), 0));
    LaunchDecode(first, m, cap ? static_cast<unsigned char *>(sink.data) : nullptr, sink, cap, frame_ends);
    CT_CUDA_CHECK(cudaEventRecord(ev_out_.get(), s));
    CT_CUDA_CHECK(cudaStreamWaitEvent(stream, ev_out_.get(), 0));
}

// ---- KITTI filter and time ranges --------------------------------------------------------------------------------------
void KittiFrameFilterDevice(int device, const cticp_device_scan &scan, const cticp_cloud_sink &sink,
                            cudaStream_t stream) {
    CT_CUDA_CHECK(cudaSetDevice(device));
    CheckFilterSink(sink, scan.num_points);
    const ScanArgs a = CheckDeviceScan(scan, device, sink.t_dtype != 0);
    if (a.n == 0) return;
    RequireDeviceRange(sink.data, SpanBytes(a.n, sink.point_step, SinkRecordWidth(sink), "sink"), device, "sink");
    LaunchFilter(device, scan, a, sink, static_cast<unsigned char *>(sink.data), stream);
}

void KittiFrameFilter(int device, const cticp_cloud_view &cloud, const cticp_cloud_sink &sink) {
    CheckFilterSink(sink, cloud.num_points);
    if (cloud.num_points == 0) return;
    const uint64_t in_bytes = CloudBytes(cloud, sink.t_dtype != 0);
    const uint64_t out_bytes = SpanBytes(cloud.num_points, sink.point_step, SinkRecordWidth(sink), "sink");
    CT_CUDA_CHECK(cudaSetDevice(device));
    cticp::Stream st(cudaStreamNonBlocking);
    cudaStream_t s = st.get();
    DeviceArray<unsigned char> in, out;
    in.reserve(in_bytes, s);
    out.reserve(out_bytes, s);
    CT_CUDA_CHECK(cudaMemcpyAsync(in.data(), cloud.data, in_bytes, cudaMemcpyHostToDevice, s));
    CT_CUDA_CHECK(cudaMemcpyAsync(out.data(), sink.data, out_bytes, cudaMemcpyHostToDevice, s));
    const cticp_device_scan scan = DeviceScanOfCloud(cloud, in.data());
    const ScanArgs a = CheckDeviceScan(scan, device, sink.t_dtype != 0);
    LaunchFilter(device, scan, a, sink, out.data(), s);
    CT_CUDA_CHECK(cudaMemcpyAsync(sink.data, out.data(), out_bytes, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
}

void ScanTimeRangesDevice(int device, const cticp_device_scan &scan, const uint64_t *frame_ends, uint64_t m,
                          double *out_minmax, cudaStream_t stream) {
    if (m && (!frame_ends || !out_minmax)) throw std::invalid_argument("null argument");
    CT_CUDA_CHECK(cudaSetDevice(device));
    const ScanArgs a = CheckDeviceScan(scan, device, true, false);
    if (m == 0) return;
    RequireAligned(frame_ends, 8, "frame_ends");
    RequireAligned(out_minmax, 8, "out_minmax");
    RequireDeviceRange(frame_ends, sizeof(uint64_t) * m, device, "frame_ends");
    RequireDeviceRange(out_minmax, sizeof(double) * 2 * m, device, "out_minmax");
    k_time_ranges<<<(int) std::min<uint64_t>(m, (uint64_t) SmCount(device) * 8), kThreads, 0, stream>>>(a, frame_ends, m,
                                                                                                        out_minmax);
    CT_CUDA_CHECK(cudaGetLastError());
}

void ScanTimeRanges(int device, const cticp_cloud_view &cloud, const uint64_t *frame_ends, uint64_t m,
                    double *out_minmax) {
    if (m && (!frame_ends || !out_minmax)) throw std::invalid_argument("null argument");
    for (uint64_t k = 0; k < m; ++k)
        if ((k && frame_ends[k] < frame_ends[k - 1]) || frame_ends[k] > cloud.num_points)
            throw std::invalid_argument("frame_ends must be non-decreasing and at most num_points");
    if (m == 0) return;
    const uint64_t in_bytes = cloud.num_points ? CloudBytes(cloud, true) : 0;
    CT_CUDA_CHECK(cudaSetDevice(device));
    cticp::Stream st(cudaStreamNonBlocking);
    cudaStream_t s = st.get();
    DeviceArray<unsigned char> in;
    DeviceArray<uint64_t> ends;
    DeviceArray<double> out;
    in.reserve(std::max<uint64_t>(in_bytes, 1), s);
    ends.reserve(m, s);
    out.reserve(2 * m, s);
    if (in_bytes) CT_CUDA_CHECK(cudaMemcpyAsync(in.data(), cloud.data, in_bytes, cudaMemcpyHostToDevice, s));
    CT_CUDA_CHECK(cudaMemcpyAsync(ends.data(), frame_ends, sizeof(uint64_t) * m, cudaMemcpyHostToDevice, s));
    ScanArgs a{};
    a.t = in.data() + cloud.t_offset;
    a.ts = cloud.point_step;
    a.n = cloud.num_points;
    a.tdt = cloud.t_dtype;
    const unsigned tsz = scan_pack::dtype_size(cloud.t_dtype);
    a.t_aligned = tsz && cloud.t_offset % tsz == 0 && cloud.point_step % tsz == 0;
    k_time_ranges<<<(int) std::min<uint64_t>(m, (uint64_t) SmCount(device) * 8), kThreads, 0, s>>>(a, ends.data(), m,
                                                                                                   out.data());
    CT_CUDA_CHECK(cudaGetLastError());
    std::vector<double> r(2 * m);
    CT_CUDA_CHECK(cudaMemcpyAsync(r.data(), out.data(), sizeof(double) * 2 * m, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    for (uint64_t k = 0; k < m; ++k)
        if (std::isnan(r[2 * k]))
            throw std::invalid_argument("frame " + std::to_string(k) + " has a NaN timestamp");
    std::copy(r.begin(), r.end(), out_minmax);
}

// ---- PLY header ----------------------------------------------------------------------------------------------------
namespace {

int PlyType(const std::string &t) {
    if (t == "char" || t == "int8") return CTICP_DTYPE_INT8;
    if (t == "uchar" || t == "uint8") return CTICP_DTYPE_UINT8;
    if (t == "short" || t == "int16") return CTICP_DTYPE_INT16;
    if (t == "ushort" || t == "uint16") return CTICP_DTYPE_UINT16;
    if (t == "int" || t == "int32") return CTICP_DTYPE_INT32;
    if (t == "uint" || t == "uint32") return CTICP_DTYPE_UINT32;
    if (t == "float" || t == "float32") return CTICP_DTYPE_FLOAT32;
    if (t == "double" || t == "float64") return CTICP_DTYPE_FLOAT64;
    return 0;
}

std::vector<std::string> Words(const std::string &line) {
    std::vector<std::string> w;
    size_t i = 0;
    while (i < line.size()) {
        while (i < line.size() && (line[i] == ' ' || line[i] == '\t' || line[i] == '\r')) ++i;
        size_t j = i;
        while (j < line.size() && line[j] != ' ' && line[j] != '\t' && line[j] != '\r') ++j;
        if (j > i) w.push_back(line.substr(i, j - i));
        i = j;
    }
    return w;
}

}  // namespace

void PlyLayoutParse(const char *bytes, uint64_t n, cticp_ply_layout *out) {
    if (!bytes || !out) throw std::invalid_argument("null argument");
    uint64_t pos = 0;
    auto next_line = [&](std::string &line) {
        const void *nl = memchr(bytes + pos, '\n', n - pos);
        if (!nl) throw std::invalid_argument("PLY: the header has no end_header line");
        const uint64_t e = static_cast<const char *>(nl) - bytes;
        line.assign(bytes + pos, e - pos);
        pos = e + 1;
    };
    std::string line;
    next_line(line);
    if (Words(line) != std::vector<std::string>{"ply"}) throw std::invalid_argument("PLY: no ply magic");
    struct Prop {
        std::string name;
        int dtype;
        uint32_t offset;
    };
    std::vector<Prop> props;
    bool format = false, in_vertex = false, seen_vertex = false;
    uint64_t count = 0;
    uint32_t step = 0;
    for (;;) {
        next_line(line);
        const std::vector<std::string> w = Words(line);
        if (w.empty() || w[0] == "comment" || w[0] == "obj_info") continue;
        if (w[0] == "end_header") break;
        if (w[0] == "format") {
            if (w.size() < 2) throw std::invalid_argument("PLY: a malformed format line");
            if (w[1] == "ascii" || w[1] == "binary_big_endian")
                throw UnsupportedError("PLY: " + w[1] + " bodies are not supported (binary_little_endian only)");
            if (w[1] != "binary_little_endian") throw std::invalid_argument("PLY: unknown format " + w[1]);
            format = true;
        } else if (w[0] == "element") {
            if (w.size() != 3) throw std::invalid_argument("PLY: a malformed element line");
            if (w[1] != "vertex") throw UnsupportedError("PLY: element " + w[1] + " (only vertex is supported)");
            if (seen_vertex) throw std::invalid_argument("PLY: two vertex elements");
            char *end = nullptr;
            errno = 0;
            count = std::strtoull(w[2].c_str(), &end, 10);
            if (errno || *end || w[2][0] == '-') throw std::invalid_argument("PLY: a malformed vertex count");
            in_vertex = seen_vertex = true;
        } else if (w[0] == "property") {
            if (!in_vertex) throw std::invalid_argument("PLY: a property outside an element");
            if (w.size() >= 2 && w[1] == "list") throw UnsupportedError("PLY: list properties are not supported");
            if (w.size() != 3) throw std::invalid_argument("PLY: a malformed property line");
            const int dt = PlyType(w[1]);
            if (!dt) throw std::invalid_argument("PLY: unknown property type " + w[1]);
            for (const Prop &p : props)
                if (p.name == w[2]) throw std::invalid_argument("PLY: property " + w[2] + " appears twice");
            props.push_back(Prop{w[2], dt, step});
            step += scan_pack::dtype_size(dt);
        } else {
            throw std::invalid_argument("PLY: unknown header line '" + line + "'");
        }
    }
    if (!format) throw std::invalid_argument("PLY: no format line");
    if (!seen_vertex) throw std::invalid_argument("PLY: no vertex element");
    auto find = [&](const char *name) -> const Prop * {
        for (const Prop &p : props)
            if (p.name == name) return &p;
        return nullptr;
    };
    const Prop *x = find("x"), *y = find("y"), *z = find("z");
    if (!x || !y || !z) throw std::invalid_argument("PLY: the vertex element lacks x, y or z");
    if (x->dtype != y->dtype || x->dtype != z->dtype)
        throw std::invalid_argument("PLY: x, y and z are of different types");
    if (x->dtype != CTICP_DTYPE_FLOAT32 && x->dtype != CTICP_DTYPE_FLOAT64)
        throw std::invalid_argument("PLY: x, y and z must be float or double");
    const uint32_t xs = scan_pack::dtype_size(x->dtype);
    if (y->offset != x->offset + xs || z->offset != y->offset + xs)
        throw std::invalid_argument("PLY: x, y and z are not consecutive");
    const Prop *t = find("timestamp");
    if (!t) t = find("t");
    if (!t) t = find("timestamps");
    if (step && count > (n - pos) / step) throw std::invalid_argument("PLY: the body is shorter than its vertex count");
    *out = cticp_ply_layout{};
    out->body_offset = pos;
    out->num_points = count;
    out->point_step = step;
    out->xyz_offset = x->offset;
    out->xyz_dtype = x->dtype;
    out->t_offset = t ? t->offset : 0;
    out->t_dtype = t ? t->dtype : 0;
}

// ---- ground truth ------------------------------------------------------------------------------------------------------
namespace {

Se3 Se3Of(const M3 &R, V3 t) { return Se3{qnormalized(qfromR(R)), t}; }   // slam::SE3(Quaterniond(R), tr)

// Eigen's AngleAxis(angle, axis) as a quaternion: (sin(angle / 2) axis, cos(angle / 2))
Q4 QAxis(double angle, int axis) {
    const double ha = 0.5 * angle, s = std::sin(ha);
    Q4 q{0.0, 0.0, 0.0, std::cos(ha)};
    (axis == 0 ? q.x : axis == 1 ? q.y : q.z) = s;
    return q;
}
Q4 QYawPitchRoll(double yaw, double pitch, double roll) {   // AngleAxis(yaw, Z) * AngleAxis(pitch, Y) * AngleAxis(roll, X)
    return qmul(qmul(QAxis(yaw, 2), QAxis(pitch, 1)), QAxis(roll, 0));
}

Se3 KittiCalib(int which) {   // kKITTITrCalibrations, dataset.cpp:52-73
    static const double R[3][9] = {
        {4.276802385584e-04, -9.999672484946e-01, -8.084491683471e-03, -7.210626507497e-03, 8.081198471645e-03,
         -9.999413164504e-01, 9.999738645903e-01, 4.859485810390e-04, -7.206933692422e-03},
        {2.347736981471e-04, -9.999441545438e-01, -1.056347781105e-02, 1.044940741659e-02, 1.056535364138e-02,
         -9.998895741176e-01, 9.999453885620e-01, 1.243653783865e-04, 1.045130299567e-02},
        {-1.857739385241e-03, -9.999659513510e-01, -8.039975204516e-03, -6.481465826011e-03, 8.051860151134e-03,
         -9.999466081774e-01, 9.999773098287e-01, -1.805528627661e-03, -6.496203536139e-03}};
    static const double T[3][3] = {{-1.198459927713e-02, -5.403984729748e-02, -2.921968648686e-01},
                                   {-2.796816941295e-03, -7.510879138296e-02, -2.721327964059e-01},
                                   {-4.784029760483e-03, -7.337429464231e-02, -3.339968064433e-01}};
    M3 m;
    for (int i = 0; i < 9; ++i) m.m[i / 3][i % 3] = R[which][i];
    return Se3Of(m, V3{T[which][0], T[which][1], T[which][2]});
}

Se3 Kitti360Calib() {   // kKITTI360_Calib, dataset.cpp:135-145
    const double R[9] = {9.999290633685804508e-01,  5.805355888196038310e-03,  1.040029024212630118e-02,
                         5.774300279226996999e-03,  -9.999787876452227442e-01, 3.013573682642321436e-03,
                         1.041756443854582707e-02, -2.953305511449066945e-03, -9.999413744330052367e-01};
    M3 m;
    for (int i = 0; i < 9; ++i) m.m[i / 3][i % 3] = R[i];
    return Se3Of(m, V3{-7.640302229235816922e-01, 2.966030253893782165e-01, -8.433819635885287935e-01});
}

// kNCLT_Calib, dataset.cpp:184-198: the matrix of a rotation built through quaternions, not renormalised
struct Mat4 {
    M3 R;
    V3 t;
};
Mat4 NcltCalib() {
    const double roll = (0.807 / 180.) * M_PI, pitch = (0.166 / 180.) * M_PI, yaw = (-90.703 / 180.) * M_PI;
    return Mat4{qtoR(QYawPitchRoll(yaw, pitch, roll)), V3{0.002, -0.004, -0.957}};
}

Se3 HiltiCalib(int dataset) {   // kHILTI_2021_Calib / kHILTI_2022_Lidar_To_Imu, dataset.cpp:215-224 (Quaterniond(w,x,y,z))
    if (dataset == CTICP_DATASET_HILTI_2021)
        return Se3{qnormalized(qnormalized(Q4{0.999993918507834, 0.0012283821413574625, -0.0032596475280467258,
                                              -0.00016947759535612024})),
                   V3{0.01001966915517371, -0.006645473484212856, 0.09473042428051345}};
    return Se3{qnormalized(qnormalized(Q4{0.7071068, -0.7071068, 0.0, 0.0})), V3{-0.001, -0.00855, 0.055}};
}

Mat4 MatOf(const Se3 &p) { return Mat4{qtoR(p.q), p.t}; }   // TSE3::Matrix(): quat.toRotationMatrix(), not normalised
Mat4 Mul(const Mat4 &a, const Mat4 &b) {
    Mat4 r;
    r.R = mmul(a.R, b.R);
    const V3 rt{a.R.m[0][0] * b.t.x + a.R.m[0][1] * b.t.y + a.R.m[0][2] * b.t.z,
                a.R.m[1][0] * b.t.x + a.R.m[1][1] * b.t.y + a.R.m[1][2] * b.t.z,
                a.R.m[2][0] * b.t.x + a.R.m[2][1] * b.t.y + a.R.m[2][2] * b.t.z};
    r.t = rt + a.t;
    return r;
}
Mat4 Inverse(const Mat4 &a) {   // of a rigid [R t; 0 1]: [R^T, -R^T t]
    Mat4 r;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) r.R.m[i][j] = a.R.m[j][i];
    const V3 v{r.R.m[0][0] * a.t.x + r.R.m[0][1] * a.t.y + r.R.m[0][2] * a.t.z,
               r.R.m[1][0] * a.t.x + r.R.m[1][1] * a.t.y + r.R.m[1][2] * a.t.z,
               r.R.m[2][0] * a.t.x + r.R.m[2][1] * a.t.y + r.R.m[2][2] * a.t.z};
    r.t = V3{-v.x, -v.y, -v.z};
    return r;
}

std::vector<std::string> Lines(const char *text, uint64_t n) {
    std::vector<std::string> lines;
    uint64_t b = 0;
    while (b < n) {
        const void *nl = memchr(text + b, '\n', n - b);
        const uint64_t e = nl ? static_cast<const char *>(nl) - text : n;
        lines.emplace_back(text + b, e - b);
        b = e + 1;
    }
    return lines;
}

// `istream >> double` over the line's whitespace-separated values into v[0..k): libstdc++'s num_get takes the longest
// prefix of the form [+-] digits [. digits] [(e|E) [+-] digits] (no nan, inf or hex) and converts it; a value without a
// digit becomes 0 and ends the line; the values after the line's end keep what they held
void ReadValues(const std::string &line, double *v, int k) {
    const char *p = line.c_str();
    auto digits = [](const char *&q) {
        const char *b = q;
        while (*q >= '0' && *q <= '9') ++q;
        return q > b;
    };
    for (int i = 0; i < k; ++i) {
        while (*p == ' ' || *p == '\t' || *p == '\r' || *p == '\v' || *p == '\f') ++p;
        if (!*p) return;
        const char *q = p;
        if (*q == '+' || *q == '-') ++q;
        bool any = digits(q);
        if (*q == '.') {
            ++q;
            any = digits(q) || any;
        }
        if (any && (*q == 'e' || *q == 'E')) {
            ++q;
            if (*q == '+' || *q == '-') ++q;
            digits(q);
        }
        if (!any) {
            v[i] = 0.0;
            return;
        }
        v[i] = std::strtod(std::string(p, q).c_str(), nullptr);
        p = q;
    }
}

}  // namespace

std::vector<cticp_pose> GroundTruthParse(int dataset, int sequence_id, const char *text, uint64_t n) {
    if (n && !text) throw std::invalid_argument("null text");
    const std::vector<std::string> lines = Lines(text, n);
    std::vector<cticp_pose> poses;
    auto pose_of = [](const Se3 &p, double t, uint32_t fid) {
        cticp_pose r{};
        r.quat[0] = p.q.x; r.quat[1] = p.q.y; r.quat[2] = p.q.z; r.quat[3] = p.q.w;
        r.tr[0] = p.t.x; r.tr[1] = p.t.y; r.tr[2] = p.t.z;
        r.ref_timestamp = 0.0;
        r.dest_timestamp = t;
        r.ref_frame_id = 0;
        r.dest_frame_id = fid;
        return r;
    };
    std::vector<Se3> raw;   // the file's poses, before transform_poses
    std::vector<double> stamps;
    Mat4 calib{M3{{{1, 0, 0}, {0, 1, 0}, {0, 0, 1}}}, V3{0, 0, 0}};
    switch (dataset) {
        case CTICP_DATASET_KITTI_RAW: case CTICP_DATASET_KITTI: case CTICP_DATASET_KITTI_360:
        case CTICP_DATASET_KITTI_CARLA: {
            if (dataset == CTICP_DATASET_KITTI || dataset == CTICP_DATASET_KITTI_RAW) {
                if (sequence_id < 0 || sequence_id > 21)
                    throw std::invalid_argument("KITTI: sequence id outside [0, 21]");
                calib = MatOf(KittiCalib(sequence_id <= 2 ? 0 : sequence_id == 3 ? 1 : 2));
            } else if (dataset == CTICP_DATASET_KITTI_360) {
                calib = MatOf(Kitti360Calib());
            }
            for (const std::string &line : lines) {   // LoadPosesKITTIFormat, io.cxx:252-279
                if (line.empty()) continue;
                double P[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
                ReadValues(line, P, 12);
                M3 R;
                for (int i = 0; i < 3; ++i)
                    for (int j = 0; j < 3; ++j) R.m[i][j] = P[4 * i + j];
                raw.push_back(Se3{qfromR(R), V3{P[3], P[7], P[11]}});
            }
            break;
        }
        case CTICP_DATASET_NCLT: {   // ReadNCLTPoses, dataset.cpp:319-381
            calib = NcltCalib();
            bool have_init = false;
            Se3 init_inv{};
            for (size_t li = 0; li < lines.size(); ++li) {
                std::string line = lines[li];
                std::vector<std::string> tokens;
                while (!line.empty()) {
                    const size_t c = line.find_first_of(',');
                    if (c == std::string::npos) {
                        tokens.push_back(line);
                        break;
                    }
                    tokens.push_back(line.substr(0, c));
                    line = line.substr(c + 1);
                }
                if (tokens.size() != 7)
                    throw std::invalid_argument("NCLT ground truth: line " + std::to_string(li + 1) + " has " +
                                                std::to_string(tokens.size()) + " values, not 7");
                double v[7];
                for (int k = 0; k < 7; ++k) {   // std::stod: leading blanks, then a number; out of range throws
                    const char *s = tokens[k].c_str();
                    char *end = nullptr;
                    errno = 0;
                    v[k] = std::strtod(s, &end);
                    if (end == s || errno == ERANGE)
                        throw std::invalid_argument("NCLT ground truth: line " + std::to_string(li + 1) +
                                                    ": a value is not a number");
                }
                const Q4 q = qfromR(qtoR(QYawPitchRoll(v[6], v[5], v[4])));
                const double nq = std::sqrt(qdot(q, q)), nt = std::sqrt(v[1] * v[1] + v[2] * v[2] + v[3] * v[3]);
                if (nq != nq || nt != nt) continue;
                const Se3 p{q, V3{v[1], v[2], v[3]}};
                if (!have_init) {
                    init_inv = se3_inverse(p);
                    have_init = true;
                }
                raw.push_back(se3_mul(init_inv, p));
                stamps.push_back(v[0]);
            }
            break;
        }
        case CTICP_DATASET_HILTI_2021: case CTICP_DATASET_HILTI_2022: {   // ReadHILTIPosesInLidarFrame, :642-677
            const Se3 l2i = HiltiCalib(dataset), i2l = se3_inverse(l2i);
            for (const std::string &line : lines) {
                double v[8] = {-1.0, 0, 0, 0, 0, 0, 0, 1};   // TPose defaults: dest_timestamp -1, identity
                ReadValues(line, v, 8);
                const Se3 p{Q4{v[4], v[5], v[6], v[7]}, V3{v[1], v[2], v[3]}};
                poses.push_back(pose_of(se3_mul(se3_mul(i2l, p), l2i), v[0], 0xFFFFFFFFu));
            }
            return poses;
        }
        default:
            throw std::invalid_argument("ground truth: unknown dataset " + std::to_string(dataset));
    }
    // transform_poses, dataset.cpp:1006-1050
    const Mat4 calib_i = Inverse(calib);   // rigid inverse; the reference's Matrix4d::inverse() agrees to ~1e-16
    for (size_t i = 0; i < raw.size(); ++i) {
        const Mat4 m = Mul(Mul(calib_i, MatOf(raw[i])), calib);
        const Se3 p{qnormalized(qfromR(m.R)), m.t};
        if (dataset == CTICP_DATASET_NCLT)
            poses.push_back(pose_of(p, stamps[i], 0xFFFFFFFFu));
        else
            poses.push_back(pose_of(p, dataset == CTICP_DATASET_KITTI_CARLA ? (double) i * 0.1 : ((double) i + 0.5) * 0.1,
                                    (uint32_t) i));
    }
    return poses;
}

}  // namespace cticp
