// world_cloud.h — slam::SamplePointsInGrid (include/SlamCore/algorithm/grid_sampling.h:12-79 of the reference) on one
// device, and its incremental form: a device-resident cloud that grows call by call and always exports what
// SamplePointsInGrid returns over every point submitted so far, in call order.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/cticp.h"
#include "cuda_owner.h"

namespace cticp {

class ContinuousTrajectory;
class Engine;

class WorldCloud {
public:
    static constexpr int kMaxPointsPerVoxel = 64;
    // refusals of the options: grid_size not finite and > 0 (std::invalid_argument), num_points_per_voxel outside
    // [0, 64] (UnsupportedError)
    static void CheckOptions(const cticp_grid_sampling_options &o);
    // capacity_voxels / capacity_points 0: the defaults of DefaultCapacity
    WorldCloud(const cticp_grid_sampling_options &o, uint64_t capacity_voxels, uint64_t capacity_points, int device);
    ~WorldCloud();
    WorldCloud(const WorldCloud &) = delete;
    WorldCloud &operator=(const WorldCloud &) = delete;

    int Device() const { return device_; }
    uint64_t NumVoxels() const { return num_voxels_; }
    uint64_t NumStored() const { return num_points_; }
    // what an export returns: every stored point, or the first max_num_points + 1 of them
    uint64_t NumPoints() const;

    // host records (traj may be null: the records are world coordinates); synchronous
    void Add(ContinuousTrajectory *traj, const cticp_cloud_view &cloud, const uint64_t *segment_ends,
             const uint32_t *segment_frame_ids, size_t num_segments, cticp_world_cloud_stats *stats);
    // device records, read after the work queued on `stream`; synchronous
    void AddDevice(ContinuousTrajectory *traj, const cticp_device_scan &scan, const uint64_t *segment_ends,
                   const uint32_t *segment_frame_ids, size_t num_segments, cticp_world_cloud_stats *stats,
                   cudaStream_t stream);
    // the last frame's CTICP_POINTS_ALL_CORRECTED world points and timestamps, device to device
    void AddOdometry(Engine &engine, cticp_world_cloud_stats *stats);
    int64_t Export(const cticp_cloud_sink &sink, uint64_t *src_index);
    int64_t ExportDevice(const cticp_cloud_sink &sink, uint64_t *src_index, cudaStream_t stream);
    void Clear();

private:
    // the key pass over m records, then rank and commit. Throws before anything changes (CapacityError included).
    void Ingest(const unsigned char *xyz, size_t xs, int xyz_dtype, const unsigned char *t, size_t ts, int t_dtype,
                uint64_t m, cticp_world_cloud_stats *stats);
    void Scan(const uint32_t *in, uint32_t *out, uint64_t n, int counter);   // exclusive; total into d_cnt_[counter]
    void EnqueueExport(unsigned char *sink_data, const cticp_cloud_sink &sink, uint64_t *d_src, uint64_t m);

    cticp_grid_sampling_options opt_;
    int device_, kp_;                     // kp_ = max(1, num_points_per_voxel): the slots of a voxel
    uint64_t cap_v_, cap_p_, table_mask_;
    uint64_t num_voxels_ = 0, num_points_ = 0, num_submitted_ = 0;
    // the owning members are released in reverse declaration order, after the destructor synchronised the stream
    cticp::Stream stream_;
    Event ev_in_, ev_out_;
    DeviceArray<ulonglong2> d_table_;     // committed voxels: {key, voxel id}, open addressing, linear probing
    DeviceArray<uint32_t> d_vcount_;      // [cap_v] points per voxel
    DeviceArray<uint32_t> d_vpts_;        // [cap_v * kp] pool index of each slot, in input order
    DeviceArray<uint32_t> d_vlo_, d_vcand_;   // [cap_v] rank scratch of the voxels already committed (0 / ~0 between calls)
    DeviceArray<double4> d_pxyzt_;        // [cap_p] pool: x, y, z, t
    DeviceArray<uint64_t> d_psrc_;        // [cap_p] pool: source index
    // per call (grow-only)
    DeviceArray<unsigned char> d_rec_;    // host records as they are
    DeviceArray<double4> d_w_;            // [m] world x, y, z, t
    DeviceArray<uint32_t> d_pv_, d_slot_, d_flag_, d_keep_, d_scan0_, d_scan1_, d_nlo_, d_ncand_;
    DeviceArray<ulonglong2> d_ltab_;      // call-local voxels: {key, first point << 32 | 0}
    DeviceArray<unsigned long long> d_desc_;
    DeviceArray<uint32_t> d_ticket_;
    DeviceArray<unsigned long long> d_cnt_;   // [0] rejected, [1] new voxels, [2] kept, [3] export offsets total
    PinnedArray<unsigned long long> h_cnt_;
    DeviceArray<uint32_t> d_off_;         // export: [cap_v] offsets of the voxels
    DeviceArray<unsigned char> d_sink_;   // export to host: the sink's records
    DeviceArray<uint64_t> d_src_out_;
};

// the default capacities of a cloud created with 0: voxels clamp(2^22 (0.2 / grid_size)^2, 2^16, 2^26), points
// voxels × max(1, num_points_per_voxel), at most 2^32 - 1
void DefaultCapacity(const cticp_grid_sampling_options &o, uint64_t *capacity_voxels, uint64_t *capacity_points);

}  // namespace cticp
