// dataset.h — dataset sequences on one device: NCLT velodyne_hits.bin packet streams indexed and decoded into scans,
// the KITTI frame filter and per-frame timestamp ranges of scans in device memory, and the host readers of PLY headers
// and ground-truth files. Semantics, quirks and refusals: include/cticp.h, "Dataset sequences".
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "../../include/cticp.h"
#include "cuda_owner.h"

namespace cticp {

class NcltHits {
public:
    // bytes: host memory (on_device = false) or device memory of `device` (ordered after `stream`); copied into the
    // handle's own buffer and indexed there. std::invalid_argument for a bad magic (its byte offset in the message),
    // a truncated packet with final, num_aggregated 0.
    NcltHits(const void *bytes, uint64_t n_bytes, uint32_t num_aggregated, bool final, int device, bool on_device,
             cudaStream_t stream);
    ~NcltHits();
    NcltHits(const NcltHits &) = delete;
    NcltHits &operator=(const NcltHits &) = delete;

    int Device() const { return device_; }
    uint64_t NumFrames() const { return frame_start_.size() - 1; }
    uint64_t NumPackets() const { return packets_; }
    uint64_t NumHits() const { return frame_start_.back(); }
    uint64_t BytesUsed() const { return bytes_used_; }
    bool Walked() const { return walked_; }   // the index came from the sequential walk, not the chain check

    void FrameInfo(uint64_t first, uint64_t m, cticp_nclt_frame *out) const;
    // frames [first, first + m) into a host sink (synchronous; returns the count) or a device sink (ordered after and
    // before `stream`, no host synchronisation; frame_ends in device memory)
    int64_t ReadFrames(uint64_t first, uint64_t m, const cticp_cloud_sink &sink, uint64_t *frame_ends);
    void ReadFramesDevice(uint64_t first, uint64_t m, const cticp_cloud_sink &sink, uint64_t *frame_ends,
                          cudaStream_t stream);

private:
    void Index(uint64_t n_bytes, uint32_t num_aggregated, bool final);
    void CheckRead(uint64_t first, uint64_t m, const cticp_cloud_sink &sink) const;
    void LaunchDecode(uint64_t first, uint64_t m, unsigned char *data, const cticp_cloud_sink &sink, uint64_t cap,
                      uint64_t *frame_ends);

    int device_;
    int sms_ = 1;
    uint64_t agg_ = 1, packets_ = 0, bytes_used_ = 0;
    bool walked_ = false;
    std::vector<uint64_t> frame_start_;          // [F + 1] the frames' first hits, then the total
    std::vector<cticp_nclt_frame> info_;    // [F]
    cticp::Stream stream_;
    Event ev_in_, ev_out_;
    DeviceArray<unsigned long long> d_bytes_;    // the stream, zero-padded to whole 8-byte words
    DeviceArray<uint64_t> d_pkt_off_;            // [packets] byte offset of each packet
    DeviceArray<uint64_t> d_hit_start_;          // [packets + 1] first hit of each packet, then the total
    DeviceArray<uint64_t> d_frame_start_;        // [F + 1]
    DeviceArray<unsigned char> d_out_;           // host path: the sink records
    DeviceArray<uint64_t> d_ends_;
};

// kitti_frame_filter on a scan in device memory into a sink in device memory (may be the scan's own records), on
// `stream`; and the same on host records through the device (synchronous)
void KittiFrameFilterDevice(int device, const cticp_device_scan &scan, const cticp_cloud_sink &sink, cudaStream_t stream);
void KittiFrameFilter(int device, const cticp_cloud_view &cloud, const cticp_cloud_sink &sink);
// per-frame (min, max) timestamps; the device variant writes NaN for a frame with a NaN timestamp, the host one throws
void ScanTimeRangesDevice(int device, const cticp_device_scan &scan, const uint64_t *frame_ends, uint64_t m,
                          double *out_minmax, cudaStream_t stream);
void ScanTimeRanges(int device, const cticp_cloud_view &cloud, const uint64_t *frame_ends, uint64_t m,
                    double *out_minmax);

// host only
void PlyLayoutParse(const char *bytes, uint64_t n, cticp_ply_layout *out);
std::vector<cticp_pose> GroundTruthParse(int dataset, int sequence_id, const char *text, uint64_t n);

}  // namespace cticp
