// synthetic.h — slam::Scene and slam::SyntheticSensorAcquisition (include/SlamCore/experimental/synthetic.h,
// src/SlamCore/experimental/synthetic.cxx of the reference) on one device: the distance of points to every primitive,
// GeneratePoints / GeneratePointsCloseToLocation and GenerateFrame of a batch of frames in one launch.
// Semantics, the draw order contract and the refusals: include/cticp.h, "Synthetic scenes and sequences".
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "../../include/cticp.h"
#include "cuda_owner.h"

namespace cticp {

class ContinuousTrajectory;

// One primitive with the constants its Distance needs, computed once on the host when the scene is created.
// Triangle: p = corners, n = Normal(), b = Barycenter(), qr / tau / perm / rank = Eigen's ColPivHouseholderQR of
// A = [p0 p1 p2] (Householder vectors below the diagonal of qr, R on and above it). Line: p[0..1], n = Direction(),
// b = Barycenter(). Sphere / ball: p[0] = centre, radius.
struct SynPrim {
    double p[3][3];
    double n[3], b[3];
    double qr[3][3];
    double tau[3];
    double radius;
    int32_t perm[3];
    int32_t rank;
    int32_t kind;   // CTICP_SYN_*
    int32_t _pad0;
};

// Eigen 3.3 / 3.4 ColPivHouseholderQR<Matrix3d>::computeInPlace of the triangle of `t`, into its qr / tau / perm / rank
void FactorTriangle(SynPrim &t);

class SyntheticScene {
public:
    static constexpr uint64_t kMaxCandidates = 0xFFFFFFFFull;   // frames × primitives × points of one call (32-bit scan)
    // flat arrays: 9 doubles per triangle, 6 per line, 4 (centre, radius) per sphere or ball; std::invalid_argument for a
    // non-finite coordinate or a negative radius. Primitive index order: triangles, lines, spheres, balls.
    SyntheticScene(const double *triangles, uint64_t nt, const double *lines, uint64_t nl, const double *spheres,
                   uint64_t ns, const double *balls, uint64_t nb, int device);
    ~SyntheticScene();
    SyntheticScene(const SyntheticScene &) = delete;
    SyntheticScene &operator=(const SyntheticScene &) = delete;

    int Device() const { return device_; }
    uint64_t NumPrimitives() const { return prims_.size(); }

    // Distance of m host points to every primitive: out[q * P + p]; synchronous
    void Distance(const double *points, uint64_t m, double *out);
    // GeneratePoints (location == nullptr) / GeneratePointsCloseToLocation(n, location, distance): fp64 xyz triples and
    // (primitive, point) pairs, min(cap, count) of each; returns the count; synchronous
    int64_t GeneratePoints(uint64_t n, const double *location, double distance, uint64_t seed, double *xyz, uint64_t cap,
                           uint32_t *src_index);
    // GenerateFrame of m frames into a host sink (returns the count; synchronous) or a device sink (ordered after and
    // before `stream`, no host synchronisation; frame_ends and src_index in device memory)
    int64_t GenerateFrames(ContinuousTrajectory &traj, const cticp_synthetic_frame *frames, uint64_t m, uint64_t n,
                           double distance, uint64_t seed, const cticp_cloud_sink &sink, uint32_t *src_index,
                           uint64_t *frame_ends);
    void GenerateFramesDevice(ContinuousTrajectory &traj, const cticp_synthetic_frame *frames, uint64_t m, uint64_t n,
                              double distance, uint64_t seed, const cticp_cloud_sink &sink, uint32_t *src_index,
                              uint64_t *frame_ends, cudaStream_t stream);

private:
    struct Plan {
        uint64_t m, n, tiles, upper;
    };
    Plan CheckFrames(const ContinuousTrajectory &traj, const cticp_synthetic_frame *frames, uint64_t m, uint64_t n,
                     double distance, const cticp_cloud_sink &sink) const;
    // the frames' begin / end poses on the scene's stream, behind the work already queued on it
    void Poses(ContinuousTrajectory &traj, const cticp_synthetic_frame *frames, uint64_t m);
    // select + generate + compact on the scene's stream; mode 0: frames, 1: every primitive, 2: close to `location`
    void Launch(int mode, const Plan &plan, double distance, const double *location, uint64_t seed,
                const cticp_synthetic_frame *frames, unsigned char *sink_data, const cticp_cloud_sink &sink,
                uint64_t sink_cap, uint32_t *src_index, uint64_t *frame_ends);

    int device_;
    int sms_ = 1, generate_ctas_per_sm_ = 1;   // the device's SMs; CTAs of k_generate resident on one
    std::vector<SynPrim> prims_;
    // the owning members are released in reverse declaration order, after the destructor synchronised the stream
    cticp::Stream stream_;
    Event ev_in_, ev_traj_, ev_out_;
    DeviceArray<SynPrim> d_prims_;
    DeviceArray<double> d_q_;                     // host queries / the frames' begin and end timestamps
    DeviceArray<double> d_dist_;
    DeviceArray<cticp_pose> d_poses_;             // [2 m] begin, end
    DeviceArray<cticp_synthetic_frame> d_frames_;
    DeviceArray<unsigned char> d_sel_;            // [m P] selection decisions
    DeviceArray<unsigned long long> d_desc_;      // [tiles + 1] look-back descriptors, then the ticket
    DeviceArray<unsigned char> d_out_;            // host path: the sink records
    DeviceArray<uint32_t> d_src_;
    DeviceArray<uint64_t> d_ends_;
};

// SyntheticSensorAcquisition::GeneratePoses(frequency): min(cap, count) poses into `out`, returns the count; synchronous
int64_t GeneratePoses(ContinuousTrajectory &traj, double frequency, cticp_pose *out, uint64_t cap);
// slam::ApplyUniformNoise of n host poses, in place; pose i draws under key (seed, noise, i)
void ApplyUniformNoise(cticp_pose *poses, uint64_t n, double scale_rot_deg, double scale_trans_m, uint64_t seed);

}  // namespace cticp
