// device_map.h — host-side owner of the device-resident voxel map (see device_map.cuh for the layout).
#pragma once
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/cticp.h"
#include "cuda_owner.h"
#include "device_map.cuh"
#include "snapshot_format.h"

namespace cticp {

struct CapacityError : std::runtime_error {
    using std::runtime_error::runtime_error;
};

struct FrameVerdict;   // frame_policy.h

#ifdef CTICP_DEBUG_TIMERS
// host side of the phase stamps (device_map.cuh); `stamps` is a kernel's stamp array (cudaGetSymbolAddress). Both do
// nothing unless the environment has CTICP_DEBUG_TIMERS; print waits for the stream.
void phase_stamps_reset(unsigned long long *stamps, cudaStream_t stream);
void phase_stamps_print(const unsigned long long *stamps, cudaStream_t stream, const char *kernel, const char *const *labels,
                        int num_labels);
#endif

class DeviceMap {
public:
    // with_normals: maintain the per-voxel normals that RadiusSearchInPlace's sensor_location filter reads (map.h:482-490)
    DeviceMap(const cticp_map_options &options, cudaStream_t stream, bool with_normals = false);

    // InsertPointCloud (map.h:153-254): world points (fp64 xyz triples) already on the device, count on the device
    // `origin` = frame_poses.front().tr of the inserted frame (orients the normals, :222-226)
    void InsertDevice(const double *d_world_xyz, const int *d_n, size_t n_upper, V3 origin = V3{0, 0, 0});
    // same from strided host memory (synchronous; used by the cticp_map_* test entry points)
    void InsertHost(const double *xyz, size_t stride_bytes, size_t n, V3 origin = V3{0, 0, 0});
    bool HasNormals() const { return with_normals_; }
    // RemoveElementsFarFromLocation (map.h:305-322)
    void RemoveFar(V3 location, double distance);
    // one cooperative launch: world points of the sub-sampled frame under the pose pair (→ d_world), RemoveFar, InsertDevice
    void UpdateFused(const float4 *d_frame, const float4 *d_frame_lo, const int *d_n, size_t n_upper, double *d_world, const Q4 &qb, const V3 &tb,
                     const Q4 &qe, const V3 &te, bool do_remove, V3 location, double max_distance, bool do_insert, V3 origin,
                     const FrameVerdict *d_verdict = nullptr);
    // d_verdict != nullptr (frame_policy.h): a SPECULATIVE launch — the pose pair, the eviction centre and whether the frame
    // is evicted / inserted at all are read from the verdict on the device (the by-value pose arguments are ignored). The
    // caller reports the outcome it read back from the verdict:
    void CommitSpeculativeInsert(bool inserted) {
        if (inserted) ++frame_count_;
    }
    void Clear();

    // counters (synchronises the stream when stale)
    const MapCounters *SyncCounters();
    // enqueue the D2H of the counters; they are valid after the caller's next stream synchronisation
    void QueueCounterReadback();
    const MapCounters *HostCounters() const { return h_counters_.data(); }
    void NotifyStreamSynchronized() { readback_pending_ = false; }
    void CheckOverflow();
    // tombstone purge / growth, driven by HostCounters(); call between frames
    void MaintainTables();
    // room for an insert of up to n_new points (grows / purges a table now if a probe sequence could wrap)
    void EnsureRoomFor(size_t n_new);

    // SearchParamsFromRadiusSearch (map.h:416-432)
    void SearchParams(double radius, int *level, int *voxel_neighborhood) const;
    const MapLevel &Level(int i) const { return levels_[i]; }
    int NumLevels() const { return (int) levels_.size(); }
    const cticp_map_options &Options() const { return options_; }
    cudaStream_t Stream() const { return stream_; }

    // GetMapPoints (map.h:354-376) in (voxel, insertion) order; returns the point count
    size_t Export(int level, std::vector<double> &xyz, std::vector<int> &voxels);

    int launches() const { return launches_; }
    int rebuilds() const { return rebuilds_; }

    // snapshots (snapshot.cu, snapshot_format.h). SnapshotMeta: capacities, device counters and frame count of every level
    // (synchronises the stream; the host copy of the counters is left alone)
    snap::MapMeta SnapshotMeta() const;
    // the map section: its header, then the packed levels with one D2H copy, and the frame origins (synchronous)
    void SaveSection(uint8_t *section, uint8_t *origins, const snap::MapMeta &meta);
    // a map section that passed snap::Validate: one H2D copy of the packed levels, then Unpack
    void LoadSection(const snap::Parsed &p);
    // pack on this map's stream, copy device to device (peer copy when the devices differ), unpack into dst on its stream
    void CloneInto(DeviceMap &dst, int src_device, int dst_device);

private:
    // the tables a MapLevel points into
    struct LevelStorage {
        DeviceArray<MapSlot> slots;
        DeviceArray<float4> points;
        DeviceArray<int> head;
        DeviceArray<double> normals;
    };
    LevelStorage AllocLevel(MapLevel &L, uint32_t cap, const cticp_resolution_param &rp);
    void RebuildLevel(size_t i, uint64_t new_cap);
    // every level's non-empty slots, point runs and normals into d_out (the map section's payload), in slot order
    void Pack(unsigned char *d_out, const snap::MapMeta &meta);
    // the payload back: every level cleared at the snapshot's capacity, each record scattered to its slot and its run to
    // slot · B; the counters and the frame origins (host or device memory) restored
    void Unpack(const unsigned char *d_payload, const snap::MapMeta &meta, const double *origins);
    void EnsureScratch(size_t n_upper);
    void EnsureFrameOrigin();

    cticp_map_options options_;
    cudaStream_t stream_;
    std::vector<MapLevel> levels_;
    std::vector<LevelStorage> storage_;   // storage_[i] owns what levels_[i] points to
    DeviceArray<MapCounters> d_counters_;
    PinnedArray<MapCounters> h_counters_;
    DeviceArray<int> d_scalar_;
    DeviceArray<int> d_next_;
    DeviceArray<uint32_t> d_touched_;
    DeviceArray<double> d_world_tmp_;
    bool dirty_ = true;
    bool readback_pending_ = false;
    bool with_normals_ = false;
    DeviceArray<double> d_frame_origins_;   // 3 doubles per frame: begin position of every inserted frame
    size_t frame_count_ = 0;
    int launches_ = 0;
    int rebuilds_ = 0;
    int fused_grid_ = 0;
};

}  // namespace cticp
