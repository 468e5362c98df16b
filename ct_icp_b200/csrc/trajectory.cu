// trajectory.cu — slam::LinearContinuousTrajectory on the device.
//
// Reference: src/SlamCore/trajectory.cxx (DoInterpolatePose :16-30, GetClosestPosesIds :54-140, TransformPoint
// :143-155, Create / CheckConsistency :164-206), include/SlamCore/types.h (GetAlphaTimestamp :192-219,
// TSE3::operator* / Interpolate :353-366, InterpolatePoseAlpha :434-452), PointCloud::RawPointsToWorldPoints
// (src/SlamCore/pointcloud.cxx:313-326).
//
// One grid-stride kernel per call, one thread per point: read the record (fp64), find the two poses around its
// timestamp, alpha, slerp + lerp, write the sink record. The two lookup indices are always equal or adjacent, so the
// acos and 1 / sin(theta) of each adjacent pair are computed once, when the trajectory is created (k_pair_consts).
#include "trajectory.h"

#include <algorithm>
#include <cmath>
#include <limits>
#include <stdexcept>
#include <string>

#include "device_checks.h"
#include "record_io.cuh"
#include "scan_pack.cuh"

namespace cticp {

namespace {

constexpr int kTrajThreads = 256;

int Blocks(size_t n) { return (int) std::max<size_t>(1, std::min<size_t>((n + kTrajThreads - 1) / kTrajThreads, 132 * 8)); }

__global__ void k_pair_consts(const cticp_pose *__restrict__ poses, int n, SlerpConsts *__restrict__ sc) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i + 1 < n; i += gridDim.x * blockDim.x) {
        const cticp_pose &a = poses[i], &b = poses[i + 1];
        sc[i] = slerp_consts(Q4{a.quat[0], a.quat[1], a.quat[2], a.quat[3]}, Q4{b.quat[0], b.quat[1], b.quat[2], b.quat[3]});
    }
}

// first index of [lo, hi) whose timestamp is not below t (std::lower_bound; hi when there is none; NaN t: lo)
__device__ __forceinline__ uint32_t lower_bound_ts(const double *__restrict__ ts, uint32_t lo, uint32_t hi, double t) {
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (__ldg(ts + mid) < t) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

struct Lookup {
    const double *ts;
    uint32_t n;
    double min_ts, max_ts;   // MinTimestamp / MaxTimestamp of Create
};

// GetClosestPosesIds with clip_on_bounds = true. by_frame: the overload with a frame id, whose poses are [a, b).
__device__ __forceinline__ void closest_poses(const Lookup &L, double t, bool by_frame, uint32_t a, uint32_t b,
                                              uint32_t &lo, uint32_t &up) {
    if (L.min_ts >= t && t >= L.max_ts) {   // the bounds check of :58, as written
        lo = up = t <= L.min_ts ? 0u : L.n - 1;
        return;
    }
    if (by_frame) {
        // lower_bound on (dest_frame_id, dest_timestamp): the poses before a compare less, those from b on do not
        up = lower_bound_ts(L.ts, a, b, t);
        if (up >= L.n) {   // past the end: the last pose carries the frame id (others are refused on the host)
            lo = up = L.n - 1;
            return;
        }
        lo = up == 0 ? 0u : up - 1;
        return;
    }
    up = lower_bound_ts(L.ts, 0, L.n, t);
    if (up >= L.n) {
        lo = up = L.n - 1;
        return;
    }
    lo = (up > 0 && __ldg(L.ts + up) > t) ? up - 1 : up;
}

// GetAlphaTimestamp of `this` = pose lo, other = pose up (min above t → 0, max below t → 0, equal timestamps → 1)
__device__ __forceinline__ double alpha_timestamp(double t, double t0, double t1) {
    const double mn = t1 < t0 ? t1 : t0, mx = t0 < t1 ? t1 : t0;
    if (mn > t) return 0.0;
    if (mx < t) return 0.0;
    if (mn == mx) return 1.0;
    return __ddiv_rn(__dsub_rn(t, mn), __dsub_rn(mx, mn));
}
// (1 - w) a + w b with the host's roundings (no FMA contraction)
__device__ __forceinline__ double lerp_rn(double a, double b, double w) {
    return __dadd_rn(__dmul_rn(__dsub_rn(1.0, w), a), __dmul_rn(w, b));
}
__device__ __forceinline__ Q4 quat_of(const cticp_pose &p) { return Q4{p.quat[0], p.quat[1], p.quat[2], p.quat[3]}; }
__device__ __forceinline__ V3 tr_of(const cticp_pose &p) { return V3{p.tr[0], p.tr[1], p.tr[2]}; }

// InterpolatePose / InterpolatePoseWithFrameId of m timestamps; range: (a, b) per query in frame-id mode, else nullptr
__global__ void __launch_bounds__(kTrajThreads) k_interpolate(const cticp_pose *__restrict__ poses,
                                                              const SlerpConsts *__restrict__ sc, Lookup L,
                                                              const double *__restrict__ qts,
                                                              const uint32_t *__restrict__ range, size_t m,
                                                              cticp_pose *__restrict__ out) {
    for (size_t i = blockIdx.x * (size_t) blockDim.x + threadIdx.x; i < m; i += (size_t) gridDim.x * blockDim.x) {
        const double t = qts[i];
        uint32_t lo, up;
        closest_poses(L, t, range != nullptr, range ? range[2 * i] : 0u, range ? range[2 * i + 1] : 0u, lo, up);
        const cticp_pose &p0 = poses[lo];
        if (lo == up) {   // DoInterpolatePose :22-23: the pose itself
            out[i] = p0;
            continue;
        }
        const cticp_pose &p1 = poses[up];
        const double alpha = alpha_timestamp(t, p0.dest_timestamp, p1.dest_timestamp);
        const Q4 q = qslerp_c(quat_of(p0), quat_of(p1), alpha, sc[lo]);   // Eigen slerp, not renormalised
        cticp_pose r;
        r.quat[0] = q.x; r.quat[1] = q.y; r.quat[2] = q.z; r.quat[3] = q.w;
        for (int k = 0; k < 3; ++k) r.tr[k] = lerp_rn(p0.tr[k], p1.tr[k], alpha);
        r.ref_timestamp = p0.ref_timestamp;
        r.dest_timestamp = lerp_rn(p0.dest_timestamp, p1.dest_timestamp, alpha);
        r.ref_frame_id = p0.ref_frame_id;
        r.dest_frame_id = p0.dest_frame_id;
        out[i] = r;
    }
}

struct SinkArgs {
    unsigned char *data;
    uint32_t step, xoff, toff;
    int xdt, tdt, x_aligned, t_aligned;
};

// RawPointsToWorldPoints: world = TransformPoint(raw, t[, frame id]) for the first m records
template <typename XT, int LOAD>
__global__ void __launch_bounds__(kTrajThreads) k_transform(const cticp_pose *__restrict__ poses,
                                                            const SlerpConsts *__restrict__ sc, Lookup L,
                                                            const unsigned char *__restrict__ xyz, size_t xs,
                                                            const unsigned char *__restrict__ t, size_t ts, int t_dtype,
                                                            int t_aligned, size_t m, const TrajSegment *__restrict__ segs,
                                                            uint32_t num_segs, SinkArgs sink) {
    for (size_t i = blockIdx.x * (size_t) blockDim.x + threadIdx.x; i < m; i += (size_t) gridDim.x * blockDim.x) {
        XT x, y, z;
        if (LOAD == kLoadVec4 && i == m - 1)   // the last record read: 12 bytes (a 16-byte load may pass the buffer)
            load_xyz<XT, kLoadNatural>(xyz + i * xs, x, y, z);
        else
            load_xyz<XT, LOAD>(xyz + i * xs, x, y, z);
        const double tt = load_timestamp(t + i * ts, t_dtype, t_aligned);
        uint32_t a = 0, b = 0;
        if (segs) {   // the segment holding point i: the first whose end lies above i
            uint32_t s0 = 0, s1 = num_segs;
            while (s0 < s1) {
                const uint32_t mid = (s0 + s1) >> 1;
                if (__ldg(&segs[mid].end) <= i) s0 = mid + 1;
                else s1 = mid;
            }
            a = __ldg(&segs[s0].a);
            b = __ldg(&segs[s0].b);
        }
        uint32_t lo, up;
        closest_poses(L, tt, segs != nullptr, a, b, lo, up);
        const V3 raw{(double) x, (double) y, (double) z};
        V3 w;
        if (lo == up) {   // TSE3::operator*: quat.normalized() * p + tr
            w = qrot(qnormalized(quat_of(poses[lo])), raw) + tr_of(poses[lo]);
        } else {
            const cticp_pose &p0 = poses[lo], &p1 = poses[up];
            const double alpha = alpha_timestamp(tt, p0.dest_timestamp, p1.dest_timestamp);
            w = ct_transform_c(quat_of(p0), tr_of(p0), quat_of(p1), tr_of(p1), alpha, raw, sc[lo]);
        }
        unsigned char *rec = sink.data + i * sink.step;
        if (sink.xdt == CTICP_DTYPE_FLOAT32) {
            store_field<float>(rec + sink.xoff, scan_pack::hi_of(w.x), sink.x_aligned);
            store_field<float>(rec + sink.xoff + 4, scan_pack::hi_of(w.y), sink.x_aligned);
            store_field<float>(rec + sink.xoff + 8, scan_pack::hi_of(w.z), sink.x_aligned);
        } else {
            store_field<double>(rec + sink.xoff, w.x, sink.x_aligned);
            store_field<double>(rec + sink.xoff + 8, w.y, sink.x_aligned);
            store_field<double>(rec + sink.xoff + 16, w.z, sink.x_aligned);
        }
        if (sink.tdt == CTICP_DTYPE_FLOAT32) store_field<float>(rec + sink.toff, scan_pack::hi_of(tt), sink.t_aligned);
        else if (sink.tdt == CTICP_DTYPE_FLOAT64) store_field<double>(rec + sink.toff, tt, sink.t_aligned);
    }
}

bool PoseLess(const cticp_pose &l, const cticp_pose &r) {   // pose_less_by_fid_and_timestamp
    return l.dest_frame_id < r.dest_frame_id || (l.dest_frame_id == r.dest_frame_id && l.dest_timestamp < r.dest_timestamp);
}

void CheckRecordDtypes(int xyz_dtype, int t_dtype) {
    if (xyz_dtype != CTICP_DTYPE_FLOAT32 && xyz_dtype != CTICP_DTYPE_FLOAT64)
        throw std::invalid_argument("x/y/z must be FLOAT32 or FLOAT64");
    if (!scan_pack::dtype_size(t_dtype)) throw std::invalid_argument("unknown timestamp dtype");
}

}  // namespace

ContinuousTrajectory::ContinuousTrajectory(const cticp_pose *poses, size_t n, int device) : device_(device) {
    if (n == 0 || !poses) throw std::invalid_argument("The trajectory created is invalid: no poses");
    if (n > (size_t) std::numeric_limits<int32_t>::max()) throw std::invalid_argument("too many poses");
    for (size_t i = 0; i < n; ++i)
        if (std::isnan(poses[i].dest_timestamp)) throw std::invalid_argument("a pose has a NaN dest_timestamp");
    poses_.assign(poses, poses + n);
    std::stable_sort(poses_.begin(), poses_.end(), PoseLess);
    // Create :169-177, including the maximum's start at numeric_limits<double>::min() (the smallest positive double)
    min_ts_ = std::numeric_limits<double>::max();
    max_ts_ = std::numeric_limits<double>::min();
    for (const auto &p : poses_) {
        if (p.dest_timestamp < min_ts_) min_ts_ = p.dest_timestamp;
        if (p.dest_timestamp > max_ts_) max_ts_ = p.dest_timestamp;
    }
    // CheckConsistency :189-206
    const uint32_t ref = poses_.front().ref_frame_id;
    for (size_t i = 1; i < n; ++i) {
        if (poses_[i].ref_frame_id != ref) throw std::invalid_argument("Inconsistent reference frames");
        if (poses_[i].dest_frame_id != poses_[i - 1].dest_frame_id &&
            !(poses_[i].dest_timestamp >= poses_[i - 1].dest_timestamp))
            throw std::invalid_argument("Inconsistent Timestamps");
    }
    CT_CUDA_CHECK(cudaSetDevice(device_));
    stream_ = cticp::Stream(cudaStreamNonBlocking);
    ev_in_ = Event(cudaEventDisableTiming);
    ev_out_ = Event(cudaEventDisableTiming);
    cudaStream_t s = stream_.get();
    d_poses_.reserve(n, s);
    d_ts_.reserve(n, s);
    d_sc_.reserve(std::max<size_t>(n - 1, 1), s);
    std::vector<double> ts(n);
    for (size_t i = 0; i < n; ++i) ts[i] = poses_[i].dest_timestamp;
    CT_CUDA_CHECK(cudaMemcpyAsync(d_poses_.data(), poses_.data(), sizeof(cticp_pose) * n, cudaMemcpyHostToDevice, s));
    CT_CUDA_CHECK(cudaMemcpyAsync(d_ts_.data(), ts.data(), sizeof(double) * n, cudaMemcpyHostToDevice, s));
    if (n > 1) {
        k_pair_consts<<<Blocks(n - 1), kTrajThreads, 0, s>>>(d_poses_.data(), (int) n, d_sc_.data());
        CT_CUDA_CHECK(cudaGetLastError());
    }
    CT_CUDA_CHECK(cudaStreamSynchronize(s));   // the host vectors the copies read go out of scope
}

ContinuousTrajectory::~ContinuousTrajectory() {
    if (stream_.get()) {
        cudaSetDevice(device_);
        cudaStreamSynchronize(stream_.get());
    }
}

void ContinuousTrajectory::FrameRange(uint32_t frame_id, uint32_t *a, uint32_t *b) const {
    auto lo = std::lower_bound(poses_.begin(), poses_.end(), frame_id,
                               [](const cticp_pose &p, uint32_t f) { return p.dest_frame_id < f; });
    auto hi = std::upper_bound(lo, poses_.end(), frame_id,
                               [](uint32_t f, const cticp_pose &p) { return f < p.dest_frame_id; });
    *a = (uint32_t) (lo - poses_.begin());
    *b = (uint32_t) (hi - poses_.begin());
}

void ContinuousTrajectory::Interpolate(const double *timestamps, const uint32_t *frame_ids, size_t m, cticp_pose *out) {
    if (m == 0) return;
    if (!timestamps || !out) throw std::invalid_argument("null argument");
    std::vector<uint32_t> range(frame_ids ? 2 * m : 0);
    if (frame_ids) {
        const uint32_t last = poses_.back().dest_frame_id;
        for (size_t i = 0; i < m; ++i) {
            const double t = timestamps[i];
            // GetClosestPosesIds :126-133: past every pose of a trajectory whose last frame is another one (a query the
            // bounds check clips never gets there)
            if (frame_ids[i] > last && !(min_ts_ >= t && t >= max_ts_))
                throw std::invalid_argument("Invalid frame or trajectory. Got request for frame " +
                                            std::to_string(frame_ids[i]) + " when max frame_id in trajectory is " +
                                            std::to_string(last));
            FrameRange(frame_ids[i], &range[2 * i], &range[2 * i + 1]);
        }
    }
    CT_CUDA_CHECK(cudaSetDevice(device_));
    cudaStream_t s = stream_.get();
    d_qts_.reserve(m, s);
    d_qout_.reserve(m, s);
    if (frame_ids) d_qrange_.reserve(2 * m, s);
    CT_CUDA_CHECK(cudaMemcpyAsync(d_qts_.data(), timestamps, sizeof(double) * m, cudaMemcpyHostToDevice, s));
    if (frame_ids)
        CT_CUDA_CHECK(cudaMemcpyAsync(d_qrange_.data(), range.data(), sizeof(uint32_t) * 2 * m, cudaMemcpyHostToDevice, s));
    const Lookup L{d_ts_.data(), (uint32_t) poses_.size(), min_ts_, max_ts_};
    k_interpolate<<<Blocks(m), kTrajThreads, 0, s>>>(d_poses_.data(), d_sc_.data(), L, d_qts_.data(),
                                                     frame_ids ? d_qrange_.data() : nullptr, m, d_qout_.data());
    CT_CUDA_CHECK(cudaGetLastError());
    CT_CUDA_CHECK(cudaMemcpyAsync(out, d_qout_.data(), sizeof(cticp_pose) * m, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
}

void ContinuousTrajectory::InterpolateDevice(const double *d_timestamps, size_t m, cticp_pose *d_out) {
    if (m == 0) return;
    CT_CUDA_CHECK(cudaSetDevice(device_));
    const Lookup L{d_ts_.data(), (uint32_t) poses_.size(), min_ts_, max_ts_};
    k_interpolate<<<Blocks(m), kTrajThreads, 0, stream_.get()>>>(d_poses_.data(), d_sc_.data(), L, d_timestamps, nullptr,
                                                                 m, d_out);
    CT_CUDA_CHECK(cudaGetLastError());
}

std::vector<TrajSegment> ContinuousTrajectory::ResolveSegments(const uint64_t *segment_ends,
                                                               const uint32_t *segment_frame_ids, size_t num_segments,
                                                               uint64_t num_points) const {
    std::vector<TrajSegment> segs;
    if (num_segments == 0) return segs;
    if (!segment_ends || !segment_frame_ids) throw std::invalid_argument("segments: null segment_ends / segment_frame_ids");
    if (num_segments > std::numeric_limits<uint32_t>::max()) throw std::invalid_argument("segments: too many");
    const uint32_t last = poses_.back().dest_frame_id;
    segs.resize(num_segments);
    for (size_t s = 0; s < num_segments; ++s) {
        if (s > 0 && segment_ends[s] < segment_ends[s - 1])
            throw std::invalid_argument("segments: segment_ends must be non-decreasing");
        // the reference CHECK-fails on such a frame for every point the bounds check does not clip: refused as a whole
        if (segment_frame_ids[s] > last)
            throw std::invalid_argument("segments: frame " + std::to_string(segment_frame_ids[s]) +
                                        " lies beyond the trajectory (max frame_id " + std::to_string(last) + ")");
        segs[s].end = segment_ends[s];
        FrameRange(segment_frame_ids[s], &segs[s].a, &segs[s].b);
    }
    if (segment_ends[num_segments - 1] != num_points)
        throw std::invalid_argument("segments: the last segment end must be the number of points");
    return segs;
}

void ContinuousTrajectory::Launch(const unsigned char *xyz, size_t xs, int xyz_dtype, const unsigned char *t, size_t ts,
                                  int t_dtype, const std::vector<TrajSegment> &segs, unsigned char *sink_data,
                                  const cticp_cloud_sink &sink, size_t m) {
    cudaStream_t s = stream_.get();
    const TrajSegment *d_segs = nullptr;
    if (!segs.empty()) {
        d_segs_.reserve(segs.size(), s);
        CT_CUDA_CHECK(cudaMemcpyAsync(d_segs_.data(), segs.data(), sizeof(TrajSegment) * segs.size(),
                                      cudaMemcpyHostToDevice, s));
        d_segs = d_segs_.data();
    }
    const size_t xsz = xyz_dtype == CTICP_DTYPE_FLOAT64 ? 8 : 4, tsz = scan_pack::dtype_size(t_dtype);
    // natural loads when every record's field is aligned to its scalar; one 16-byte load for (N, 4)-like float32 rows
    const bool x_nat = (reinterpret_cast<uintptr_t>(xyz) % xsz) == 0 && xs % xsz == 0;
    const bool x_vec4 = xsz == 4 && (reinterpret_cast<uintptr_t>(xyz) % 16) == 0 && xs % 16 == 0;
    const int t_al = ((reinterpret_cast<uintptr_t>(t) % tsz) == 0 && ts % tsz == 0) ? 1 : 0;
    const size_t osz = sink.xyz_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8, otsz = sink.t_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8;
    SinkArgs sa;
    sa.data = sink_data;
    sa.step = sink.point_step;
    sa.xoff = sink.xyz_offset;
    sa.toff = sink.t_offset;
    sa.xdt = sink.xyz_dtype;
    sa.tdt = sink.t_dtype;
    sa.x_aligned = ((reinterpret_cast<uintptr_t>(sink_data) + sink.xyz_offset) % osz == 0 && sink.point_step % osz == 0) ? 1 : 0;
    sa.t_aligned = ((reinterpret_cast<uintptr_t>(sink_data) + sink.t_offset) % otsz == 0 && sink.point_step % otsz == 0) ? 1 : 0;
    const Lookup L{d_ts_.data(), (uint32_t) poses_.size(), min_ts_, max_ts_};
    const uint32_t ns = (uint32_t) segs.size();
    if (xsz == 8) {
        auto k = x_nat ? k_transform<double, kLoadNatural> : k_transform<double, kLoadBytes>;
        k<<<Blocks(m), kTrajThreads, 0, s>>>(d_poses_.data(), d_sc_.data(), L, xyz, xs, t, ts, t_dtype, t_al, m, d_segs, ns, sa);
    } else {
        auto k = x_vec4 ? k_transform<float, kLoadVec4>
                 : x_nat ? k_transform<float, kLoadNatural> : k_transform<float, kLoadBytes>;
        k<<<Blocks(m), kTrajThreads, 0, s>>>(d_poses_.data(), d_sc_.data(), L, xyz, xs, t, ts, t_dtype, t_al, m, d_segs, ns, sa);
    }
    CT_CUDA_CHECK(cudaGetLastError());
}

int64_t ContinuousTrajectory::Transform(const cticp_cloud_view &c, const uint64_t *segment_ends,
                                        const uint32_t *segment_frame_ids, size_t num_segments,
                                        const cticp_cloud_sink &sink) {
    const uint64_t n = c.num_points;
    if (n && !c.data) throw std::invalid_argument("cloud: null data");
    CheckRecordDtypes(c.xyz_dtype, c.t_dtype);
    const uint64_t xw = (uint64_t) c.xyz_offset + 3 * (c.xyz_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8);
    const uint64_t tw = (uint64_t) c.t_offset + scan_pack::dtype_size(c.t_dtype);
    if (xw > c.point_step || tw > c.point_step)
        throw std::invalid_argument("cloud view: a field lies outside the record (point_step)");
    const std::vector<TrajSegment> segs = ResolveSegments(segment_ends, segment_frame_ids, num_segments, n);
    if (!sink.world) throw std::invalid_argument("sink: world must be set (a trajectory writes world coordinates)");
    const size_t m = std::min<uint64_t>(sink.capacity_points, n);
    if (m == 0 || !sink.data) return (int64_t) n;
    CheckSink(sink);
    const uint64_t in_bytes = SpanBytes(m, c.point_step, std::max(xw, tw), "cloud");
    const uint64_t out_bytes = SpanBytes(m, sink.point_step, SinkRecordWidth(sink), "sink");
    CT_CUDA_CHECK(cudaSetDevice(device_));
    cudaStream_t s = stream_.get();
    d_in_.reserve(in_bytes, s);
    d_out_.reserve(out_bytes, s);
    // the records and the sink go over as they are: the bytes of the sink records outside x, y, z and t stay the caller's
    CT_CUDA_CHECK(cudaMemcpyAsync(d_in_.data(), c.data, in_bytes, cudaMemcpyHostToDevice, s));
    CT_CUDA_CHECK(cudaMemcpyAsync(d_out_.data(), sink.data, out_bytes, cudaMemcpyHostToDevice, s));
    Launch(d_in_.data() + c.xyz_offset, c.point_step, c.xyz_dtype, d_in_.data() + c.t_offset, c.point_step, c.t_dtype, segs,
           d_out_.data(), sink, m);
    CT_CUDA_CHECK(cudaMemcpyAsync(sink.data, d_out_.data(), out_bytes, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    return (int64_t) n;
}

int64_t ContinuousTrajectory::TransformDevice(const cticp_device_scan &scan, const uint64_t *segment_ends,
                                              const uint32_t *segment_frame_ids, size_t num_segments,
                                              const cticp_cloud_sink &sink, cudaStream_t stream) {
    const uint64_t n = scan.num_points;
    if (n && (!scan.xyz || !scan.t)) throw std::invalid_argument("scan: null xyz / t");
    CheckRecordDtypes(scan.xyz_dtype, scan.t_dtype);
    const std::vector<TrajSegment> segs = ResolveSegments(segment_ends, segment_frame_ids, num_segments, n);
    if (!sink.world) throw std::invalid_argument("sink: world must be set (a trajectory writes world coordinates)");
    const size_t m = std::min<uint64_t>(sink.capacity_points, n);
    if (m == 0 || !sink.data) return (int64_t) n;
    CheckSink(sink);
    CT_CUDA_CHECK(cudaSetDevice(device_));
    const uint64_t xsz = scan.xyz_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8, tsz = scan_pack::dtype_size(scan.t_dtype);
    RequireDeviceRange(scan.xyz, SpanBytes(n, scan.xyz_stride_bytes, 3 * xsz, "xyz"), device_, "xyz");
    RequireDeviceRange(scan.t, SpanBytes(n, scan.t_stride_bytes, tsz, "t"), device_, "t");
    RequireDeviceRange(sink.data, SpanBytes(m, sink.point_step, SinkRecordWidth(sink), "sink"), device_, "sink");
    cudaStream_t s = stream_.get();
    // ordered both ways with the caller's stream: behind what it queued before (the records, the sink's allocation),
    // ahead of what it queues next
    CT_CUDA_CHECK(cudaEventRecord(ev_in_.get(), stream));
    CT_CUDA_CHECK(cudaStreamWaitEvent(s, ev_in_.get(), 0));
    Launch(static_cast<const unsigned char *>(scan.xyz), scan.xyz_stride_bytes, scan.xyz_dtype,
           static_cast<const unsigned char *>(scan.t), scan.t_stride_bytes, scan.t_dtype, segs,
           static_cast<unsigned char *>(sink.data), sink, m);
    CT_CUDA_CHECK(cudaEventRecord(ev_out_.get(), s));
    CT_CUDA_CHECK(cudaStreamWaitEvent(stream, ev_out_.get(), 0));
    return (int64_t) n;
}

}  // namespace cticp
