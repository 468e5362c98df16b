// trajectory.h — slam::LinearContinuousTrajectory on one device (include/SlamCore/trajectory.h:28-130 of the reference):
// a sorted list of poses, the pose at any timestamp, and RawPointsToWorldPoints (src/SlamCore/pointcloud.cxx:313-326)
// over caller-owned point records in host or device memory.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "../../include/cticp.h"
#include "cuda_owner.h"
#include "se3.cuh"

namespace cticp {

// one segment of a transform in frame-id mode: points [previous end, end) of the frame whose poses are [a, b)
struct TrajSegment {
    uint64_t end;
    uint32_t a, b;
};

class ContinuousTrajectory {
public:
    // LinearContinuousTrajectory::Create (trajectory.cxx:164-206): sorts by (dest_frame_id, dest_timestamp), stable;
    // throws std::invalid_argument where CheckConsistency would fail, and for a NaN dest_timestamp
    ContinuousTrajectory(const cticp_pose *poses, size_t n, int device);
    ~ContinuousTrajectory();
    ContinuousTrajectory(const ContinuousTrajectory &) = delete;
    ContinuousTrajectory &operator=(const ContinuousTrajectory &) = delete;

    int Device() const { return device_; }
    const std::vector<cticp_pose> &Poses() const { return poses_; }
    double MinTimestamp() const { return min_ts_; }
    double MaxTimestamp() const { return max_ts_; }

    // InterpolatePose (frame_ids == nullptr) / InterpolatePoseWithFrameId of m host timestamps; synchronous
    void Interpolate(const double *timestamps, const uint32_t *frame_ids, size_t m, cticp_pose *out);
    // RawPointsToWorldPoints of host records into a host sink (synchronous) / of device records into a device sink (ordered
    // after and before `stream`, no host synchronisation). Return the number of points; write min(capacity, count).
    int64_t Transform(const cticp_cloud_view &cloud, const uint64_t *segment_ends, const uint32_t *segment_frame_ids,
                      size_t num_segments, const cticp_cloud_sink &sink);
    int64_t TransformDevice(const cticp_device_scan &scan, const uint64_t *segment_ends,
                            const uint32_t *segment_frame_ids, size_t num_segments, const cticp_cloud_sink &sink,
                            cudaStream_t stream);

private:
    // the segments resolved to pose ranges; empty = timestamp mode. Throws before anything is enqueued.
    std::vector<TrajSegment> ResolveSegments(const uint64_t *segment_ends, const uint32_t *segment_frame_ids,
                                             size_t num_segments, uint64_t num_points) const;
    // [a, b): the poses of frame `frame_id` (a == b where it would sort when absent)
    void FrameRange(uint32_t frame_id, uint32_t *a, uint32_t *b) const;
    void Launch(const unsigned char *xyz, size_t xs, int xyz_dtype, const unsigned char *t, size_t ts, int t_dtype,
                const std::vector<TrajSegment> &segs, unsigned char *sink_data, const cticp_cloud_sink &sink, size_t m);

    int device_;
    std::vector<cticp_pose> poses_;
    double min_ts_, max_ts_;
    // the owning members are released in reverse declaration order, after the destructor synchronised the stream
    cticp::Stream stream_;
    Event ev_in_, ev_out_;
    DeviceArray<cticp_pose> d_poses_;
    DeviceArray<double> d_ts_;
    DeviceArray<SlerpConsts> d_sc_;      // pair i: poses i and i + 1
    DeviceArray<TrajSegment> d_segs_;
    DeviceArray<double> d_qts_;          // Interpolate: the queries, their frames' pose ranges and the poses out
    DeviceArray<uint32_t> d_qrange_;
    DeviceArray<cticp_pose> d_qout_;
    DeviceArray<unsigned char> d_in_, d_out_;   // Transform: the records and the sink, copied as they are
};

}  // namespace cticp
