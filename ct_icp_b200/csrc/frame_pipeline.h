// frame_pipeline.h — device buffers and kernels of one scan's journey: pinned staging → raw float4 → sub-sampled
// frame → keypoints → world-space frame (for the map). See frame_pipeline.cu.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "device_map.h"
#include "se3.cuh"

namespace cticp {

// what k_scan_reduce leaves in device memory and in mapped pinned memory (FramePipeline::PackFromDevice)
struct ScanReduceOut {
    double t_min, t_max;
    int needs_lo;
    unsigned seq;
};
struct ScanPartial;   // frame_pipeline.cu

class FramePipeline {
public:
    FramePipeline(size_t max_points, cudaStream_t stream);

    // pinned staging buffer the host packs (x, y, z, alpha) into, then Upload(n) enqueues the H2D copy
    float4 *Staging() { return h_stage_.data(); }
    // residual planes (value - (double)(float)value, see load_raw in se3.cuh) — allocated on first use: float32 scans,
    // what LiDAR drivers emit, never need them. raw_lo: the scan as uploaded; frame_lo: the sub-sampled frame and the
    // keypoints drawn from it (also set by DistortFrame, whose output is not float32-representable).
    void EnsureLo();
    // the device lo planes only (raw, frame, keypoints, scratch): what a scan packed on the device needs
    void EnsureDeviceLo();
    float4 *StagingLo() { EnsureLo(); return h_stage_lo_.data(); }
    const float4 *StagingLoIfAny() const { return raw_lo_ ? h_stage_lo_.data() : nullptr; }
    void UploadLo(size_t n);                                  // after Upload*/UploadBegin of the same scan
    bool raw_has_lo() const { return raw_lo_; }
    bool frame_has_lo() const { return frame_lo_; }
    bool frame_distorted() const { return distorted_; }
    const float4 *d_raw_lo() const { return raw_lo_ ? raw_lo_ptr_ : nullptr; }
    const float4 *d_frame_lo() const { return frame_lo_ ? d_frame_lo_.data() : nullptr; }
    const float4 *d_keypoints_lo() const { return frame_lo_ ? d_kp_lo_.data() : nullptr; }
    size_t MaxPoints() const { return max_points_; }
    void Upload(size_t n);
    // the same copy in pieces, so that it can start while the tail of the scan is still being packed:
    // UploadBegin(n), then UploadRange over a partition of [0, n) in any order
    void UploadBegin(size_t n);
    void UploadRange(size_t begin, size_t end);
    // scan already packed and resident in HBM: read in place (no copy) until the next Upload* — the caller keeps d_src /
    // d_src_lo alive until then, or until DetachRaw()
    void UploadFromDevice(const float4 *d_src, const float4 *d_src_lo, size_t n);
    // copy a scan read in place into the pipeline's own buffers (before the caller frees it); stream-ordered
    void DetachRaw();
    // A scan in device memory (x, y, z of xyz_dtype at xyz, one t_dtype timestamp at t, both strided in bytes; the caller
    // validated the layout): two launches on the pipeline's stream. k_scan_reduce: timestamp min / max and, for float64
    // x, y, z, whether the scan needs its residual plane, to device memory and to mapped pinned memory. k_scan_pack: the
    // (x, y, z, alpha) planes into the pipeline's own raw buffers, alpha w.r.t. pose_ts = the initial estimate's {begin,
    // end} dest_timestamp, or (nullptr) the reduce's min / max read on the device.
    void PackFromDevice(const void *xyz, size_t xyz_stride, int xyz_dtype, const void *t, size_t t_stride, int t_dtype,
                        size_t n, const double *pose_ts);
    // the reduce's min / max (waits for k_scan_reduce only; the pack may still run)
    void WaitScanReduce(double *t_min, double *t_max);
    // m points of one of the summary's vectors into records in device memory (cticp_odometry_write_points_device), on
    // the pipeline's stream; mn / mx: the pose pair's timestamps ordered
    void WritePointsDevice(const float4 *pts, const float4 *lo, const double *world, size_t m, const cticp_cloud_sink &sink,
                           double mn, double mx);

    // Odometry::InitializeFrame: shuffle → sub_sample_frame → (frames 0,1: timestamp := end) → shuffle
    void SubSampleFrame(double voxel_size, uint64_t seed, uint64_t counter1, uint64_t counter2, bool override_alpha,
                        float alpha_value);
    // both of the above (GRID sampling, no truncation) in one cooperative launch
    void SampleFused(double voxel_size, double sample_voxel_size, uint64_t seed, uint64_t counter1, uint64_t counter2,
                     bool override_alpha, float alpha_value);
    // TryRegister: grid_sampling | NONE, then the optional max_num_keypoints shuffle-truncate
    void SampleKeypoints(int sampling, double sample_voxel_size, int max_num_keypoints, uint64_t seed, uint64_t counter,
                         const cticp_adaptive_options *adaptive = nullptr);
    // AdaptiveSamplePointsInGrid (include/ct_icp/algorithm/sampling.h:55-110)
    void AdaptiveSelect(const cticp_adaptive_options &o, const float4 *in, const float4 *in_lo, const uint32_t *in_src,
                        const int *d_n_in, size_t n_upper, float4 *out, float4 *out_lo, uint32_t *out_src, int *d_n_out);
    // DistortFrame (odometry.cpp:161-168) on the sub-sampled frame, in place
    void DistortFrame(const Q4 &qb, const V3 &tb, const Q4 &qe, const V3 &te);
    // world points of the sub-sampled frame / of every input point with the final pose pair
    void TransformFrame(const Q4 &qb, const V3 &tb, const Q4 &qe, const V3 &te);
    // (stream: nullptr = the pipeline's own; the egress of the summary vectors runs on a second stream)
    void TransformAll(const Q4 &qb, const V3 &tb, const Q4 &qe, const V3 &te, cudaStream_t stream = nullptr);
    void TransformInto(const float4 *pts, const float4 *lo, const int *d_n, const Q4 &qb, const V3 &tb, const Q4 &qe,
                       const V3 &te, double *d_world, cudaStream_t stream = nullptr);
    void EnsureAllWorld();

    void QueueCountsReadback();   // h_counts()[0..2] = N, F, K after the next stream sync
    const int *h_counts() const { return h_counts_.data(); }
    // the same four counters, brought back by another route (the frame verdict, frame_policy.h)
    void SetHostCounts(const int *c) {
        for (int i = 0; i < 4; ++i) h_counts_.data()[i] = c[i];
    }
    const int *d_counts() const { return d_counts_.data(); }

    const float4 *d_raw() const { return raw_ptr_; }
    const float4 *d_frame() const { return d_frame_.data(); }
    const float4 *d_keypoints() const { return d_keypoints_.data(); }
    float4 *d_keypoints_mut() { return d_keypoints_.data(); }
    const uint32_t *d_frame_src() const { return d_frame_src_.data(); }
    const uint32_t *d_keypoints_src() const { return d_kp_src_.data(); }
    const double *d_frame_world() const { return d_frame_world_.data(); }
    const double *d_all_world() const { return d_all_world_.data(); }
    int *d_count_n() { return d_counts_.data() + 0; }
    int *d_count_frame() { return d_counts_.data() + 1; }
    int *d_count_keypoints() { return d_counts_.data() + 2; }
    size_t n() const { return n_; }
    size_t h2d_bytes() const { return h2d_bytes_; }
    int launches() const { return launches_; }

    // generic "first-seen per voxel" selection (also behind cticp_grid_sample_indices)
    void GridSelect(const float4 *in, const float4 *in_lo, const uint32_t *in_src, const int *d_n_in, size_t n_upper,
                    double voxel_size, int use_perm1, uint64_t seed, uint64_t c1, int use_perm2, uint64_t c2,
                    int override_alpha, float alpha_value, float4 *out, float4 *out_lo, uint32_t *out_src, int *d_n_out);
    float4 *d_frame_lo_mut() { EnsureLo(); return d_frame_lo_.data(); }
    double *d_frame_world_mut() { return d_frame_world_.data(); }
    float4 *d_frame_mut() { return d_frame_.data(); }
    uint32_t *d_frame_src_mut() { return d_frame_src_.data(); }

private:
    int Blocks(size_t n) const;
    void BeginScan(size_t n);
    // N of a new scan reaches counts[0] as an argument of the first kernel that reads it (no 4-byte H2D copy in front of
    // the sampler): n_ when d_n is counts[0] and that kernel has not been launched yet for this scan, else -1
    int TakeHostN(const int *d_n);

    cudaStream_t stream_;
    size_t max_points_, n_ = 0, h2d_bytes_ = 0;
    bool n_on_device_ = true;
    const float4 *raw_ptr_ = nullptr, *raw_lo_ptr_ = nullptr;   // the scan being read: d_raw_ / d_raw_lo_ or a staged scan
    uint32_t grid_cap_ = 0;
    PinnedArray<float4> h_stage_;
    PinnedArray<int> h_counts_;
    DeviceArray<float4> d_raw_, d_frame_, d_keypoints_, d_tmp_points_;
    PinnedArray<float4> h_stage_lo_;
    DeviceArray<float4> d_raw_lo_, d_frame_lo_, d_kp_lo_, d_tmp_lo_;
    bool raw_lo_ = false, frame_lo_ = false, distorted_ = false;
    DeviceArray<uint32_t> d_frame_src_, d_kp_src_, d_tmp_src_;
    DeviceArray<unsigned long long> d_grid_;
    DeviceArray<int> d_slot_of_;
    DeviceArray<uint32_t> d_src_, d_win_;   // point of each position / compacted winners before the second shuffle
    DeviceArray<unsigned long long> d_desc_;   // look-back descriptors of the selections (frame_pipeline.cu)
    DeviceArray<int> d_counts_;
    DeviceArray<double> d_frame_world_, d_all_world_;
    DeviceArray<unsigned long long> d_grid2_;   // hash grid of the fused sampler's second selection
    int fused_grid_ = 0;
    // k_sample_fused leaves the hash grid clean for the next frame (CTICP_SAMPLE_PRECLEAR=0: every launch clears it itself):
    // the capacity that is clean right now
    bool preclear_ = true;
    uint32_t clean_cap_ = 0;
    DeviceArray<uint32_t> d_adaptive_;   // tile counters + flags + src of the band-major position space
    // k_scan_reduce: per-CTA partials, the last CTA's ticket, the result (device / mapped pinned, sequence number last)
    DeviceArray<ScanPartial> d_scan_partials_;
    DeviceArray<unsigned> d_scan_ticket_;
    DeviceArray<ScanReduceOut> d_scan_reduce_;
    PinnedArray<ScanReduceOut> h_scan_reduce_{cudaHostAllocMapped};
    ScanReduceOut *h_scan_reduce_dev_ = nullptr;
    unsigned scan_reduce_seq_ = 0;
    bool scan_xyz_f64_ = false;
    void EnsureScanReduce();
    int launches_ = 0;
};

}  // namespace cticp
