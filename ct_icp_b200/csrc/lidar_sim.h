// lidar_sim.h — a spinning LiDAR ray-cast on one device: a scene of a ground plane, axis-aligned boxes (solid or porous)
// and vertical cylinders, the range of given rays, and sweeps of a sensor moving along a continuous trajectory.
// Semantics, the noise key and the refusals: include/cticp.h, "Spinning-LiDAR sweeps".
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "../../include/cticp.h"
#include "cuda_owner.h"

namespace cticp {

class ContinuousTrajectory;

// the uniform xy grid the primitives are binned into: cell (ix, iy) covers [x0 + ix cell, x0 + (ix + 1) cell) ×
// [y0 + iy cell, ...), index iy nx + ix; zmax bounds every primitive's top
struct LidarGrid {
    double x0, y0, x1, y1, cell, inv_cell, zmax;
    int32_t nx, ny;
};

class LidarScene {
public:
    static constexpr uint64_t kMaxRays = 0xFFFFFFFFull;   // rays of one sweep call (32-bit scan and ray indices)
    // boxes: nb × 7 (x0 y0 z0 x1 y1 z1 mean_free_path), cylinders: nc × 4 (cx cy r h); std::invalid_argument for a
    // non-finite value, x0 > x1 (or y, z), r < 0 or a negative free path. Bins the primitives on the device.
    LidarScene(const double *boxes, uint64_t nb, const double *cylinders, uint64_t nc, bool ground, int device);
    ~LidarScene();
    LidarScene(const LidarScene &) = delete;
    LidarScene &operator=(const LidarScene &) = delete;

    int Device() const { return device_; }
    uint64_t NumBoxes() const { return nb_; }
    uint64_t NumCylinders() const { return nc_; }
    uint64_t NumCells() const { return (uint64_t) grid_.nx * (uint64_t) grid_.ny; }
    uint64_t NumCellEntries() const { return entries_; }

    // the range of n rays (fp64 xyz triples): host arrays, synchronous / device arrays, ordered after and before `stream`
    void Raycast(const double *origins, const double *directions, uint64_t n, double max_range, uint64_t seed,
                 double *out);
    void RaycastDevice(const double *origins, const double *directions, uint64_t n, double max_range, uint64_t seed,
                       double *out, cudaStream_t stream);
    // m sweeps into a host sink (returns the count; synchronous) or a device sink (ordered after and before `stream`, no
    // host synchronisation; ray_index and frame_ends in device memory)
    int64_t GenerateSweeps(ContinuousTrajectory &traj, const cticp_lidar_sensor &sensor, const cticp_lidar_frame *frames,
                           uint64_t m, uint64_t seed, const cticp_cloud_sink &sink, uint32_t *ray_index,
                           uint64_t *frame_ends);
    void GenerateSweepsDevice(ContinuousTrajectory &traj, const cticp_lidar_sensor &sensor,
                              const cticp_lidar_frame *frames, uint64_t m, uint64_t seed, const cticp_cloud_sink &sink,
                              uint32_t *ray_index, uint64_t *frame_ends, cudaStream_t stream);

private:
    struct Plan {
        uint64_t m, rays, chunks, tiles, upper;
    };
    Plan CheckSweeps(const ContinuousTrajectory &traj, const cticp_lidar_sensor &sensor, const cticp_lidar_frame *frames,
                     uint64_t m, const cticp_cloud_sink &sink) const;
    // the direction tables (host libm), the column timestamps and the trajectory's poses at them, on the scene's stream
    void Columns(ContinuousTrajectory &traj, const cticp_lidar_sensor &sensor, const cticp_lidar_frame *frames,
                 uint64_t m);
    void LaunchSweeps(const Plan &plan, const cticp_lidar_sensor &sensor, uint64_t seed, unsigned char *sink_data,
                      const cticp_cloud_sink &sink, uint64_t cap, uint32_t *ray_index, uint64_t *frame_ends);
    void LaunchRaycast(const double *o, const double *d, uint64_t n, double max_range, uint64_t seed, double *out);

    int device_;
    uint64_t nb_, nc_, entries_ = 0;
    bool ground_;
    LidarGrid grid_{};
    int sms_ = 1, sweep_ctas_per_sm_ = 1;
    // the owning members are released in reverse declaration order, after the destructor synchronised the stream
    cticp::Stream stream_;
    Event ev_in_, ev_traj_, ev_out_;
    DeviceArray<double> d_boxes_;                 // nb × 8: the 7 values and a pad (64-byte records)
    DeviceArray<double> d_cyl_;                   // nc × 4
    DeviceArray<uint2> d_cells_;                  // per cell: (start, count) in d_items_
    DeviceArray<uint32_t> d_items_;               // primitive ids, cell by cell: box b = b, cylinder c = nb + c
    DeviceArray<double> d_o_, d_d_, d_r_;         // host raycast: rays and ranges
    DeviceArray<double> d_trig_;                  // cos el, sin el (rings), cos az, sin az (columns)
    DeviceArray<double> d_ts_;                    // [m × n_azimuth] column timestamps
    DeviceArray<cticp_pose> d_poses_;             // [m × n_azimuth] the poses at them
    DeviceArray<cticp_lidar_frame> d_frames_;
    DeviceArray<unsigned long long> d_desc_;      // [tiles + 1] look-back descriptors, then the ticket
    DeviceArray<unsigned char> d_out_;            // host path: the sink records
    DeviceArray<uint32_t> d_idx_;
    DeviceArray<uint64_t> d_ends_;
};

}  // namespace cticp
