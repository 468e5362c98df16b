// engine.h — host orchestration of one odometry instance: the H100-native ct_icp::Odometry.
//
// Mirrors the control flow of src/ct_icp/odometry.cpp (RegisterFrame :199-214, InitializeMotion :276-330,
// InitializeFrame :333-382, DoRegister :386-501, TryRegister :525-601, AssessRegistration :604-684,
// RobustRegistration :780-852, UpdateMap :855-953) while every O(N)/O(K·S) stage runs on the device.
#pragma once
#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <exception>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>
#include <string>
#include <vector>

#include "../../include/cticp.h"
#include "device_map.h"
#include "frame_pipeline.h"
#include "icp.h"
#include "frame_policy.h"

namespace cticp {

struct UnsupportedError : std::runtime_error {
    using std::runtime_error::runtime_error;
};
struct TimestampError : std::runtime_error {
    using std::runtime_error::runtime_error;
};

struct HostPose {   // slam::TPose<double>
    Se3 pose = se3_identity();
    double ref_timestamp = 0, dest_timestamp = -1;
    uint32_t ref_frame_id = 0, dest_frame_id = uint32_t(-1);
};
struct HostFrame {   // ct_icp::TrajectoryFrame
    HostPose begin_pose, end_pose;
};

// A borrowed scan: x,y,z contiguous of one scalar type at `xyz`, one timestamp scalar at `t`, both strided in bytes.
// What the reference reads through XYZConst<double>() / TimestampsProxy<double>() (odometry.cpp:335-336): any source
// scalar type, converted with static_cast<double> by the proxy (include/SlamCore/data/view.h:99-120).
struct ScanView {
    const void *xyz = nullptr;
    size_t xyz_stride = 0;
    int xyz_dtype = CTICP_DTYPE_FLOAT64;   // FLOAT32 / FLOAT64
    const void *t = nullptr;
    size_t t_stride = 0;
    int t_dtype = CTICP_DTYPE_FLOAT64;     // any CTICP_DTYPE_*
    size_t n = 0;
    // in device memory of the engine's device (cticp_odometry_register_device): packed on the device after `producer`'s
    // work, instead of on the host
    bool on_device = false;
    cudaStream_t producer = nullptr;
};

// host_pack.cpp: (x, y, z, alpha) packing of points [b, e) of a contiguous float64 scan with AVX2; b a multiple of 4.
// *any_lo is set when some coordinate is not float32-representable (never cleared).
bool HostPackHasAvx2();
void PackBlockF64Avx2(const double *xyz, const double *t, size_t b, size_t e, double mn, double inv, bool spans, float4 *dst,
                      bool *any_lo);

// Minimal fork-join pool for the host passes over a scan (timestamp min/max, float4 packing): the only O(N) host
// work of RegisterFrame. After a job the workers keep polling for the next one for ~1 ms before they go to sleep on a
// condition variable (what OpenMP runtimes do by default, cf. GOMP_SPINCOUNT): when frames arrive back to back the
// team starts within a microsecond instead of a futex wake-up per worker; at sensor rate (10-20 Hz) the polling is a
// ~1 % duty cycle. The caller polls for completion as well (the job is a few tens of microseconds long).
struct CallbackError : std::runtime_error {
    using std::runtime_error::runtime_error;
};

class HostPool {
public:
    explicit HostPool(int threads);
    ~HostPool();
    int size() const { return (int) workers_.size() + 1; }
    // number of parts a pass over n items is split into (1 below the threading threshold)
    int PartsFor(size_t n) const { return (size() == 1 || n < 16384) ? 1 : size(); }
    // fn(part, parts) on every thread of the team at once (parts = PartsFor(n)); the caller runs part 0. All parts run
    // concurrently, so fn may synchronise its parts (TeamBarrier)
    void ParallelRegion(size_t n, const std::function<void(int, int)> &fn);
    // fn(begin, end, part) over [0, n) split into PartsFor(n) contiguous parts
    void ParallelFor(size_t n, const std::function<void(size_t, size_t, int)> &fn);

private:
    void Worker(int id);
    std::vector<std::thread> workers_;
    std::mutex mu_;
    std::condition_variable cv_start_;
    const std::function<void(int, int)> *fn_ = nullptr;
    std::atomic<uint64_t> generation_{0};
    std::atomic<int> pending_{0};
    bool stop_ = false;
};

class Engine {
    struct FrameInfo {
        int registered_fid = -1;
        uint32_t frame_id = uint32_t(-1);
        double begin_timestamp = -1, end_timestamp = -1;
    };
    struct Summary {   // RegistrationSummary minus the point vectors
        HostFrame frame, initial_frame;
        int sample_size = 0, number_of_residuals = 0, robust_level = 0;
        double distance_correction = 0, relative_distance = 0, relative_orientation = 0, ego_orientation = 0;
        bool success = true, points_added = false;
        int number_of_attempts = 0;
        std::string error_message;
        cticp_icp_summary icp{};
        double t_try_register = 0, t_sampling = 0;
    };
    struct MotionModel {
        bool present = false;
        cticp_motion_model_options options{};
        HostFrame previous_frame;
    };

public:
    Engine(const cticp_odometry_options &options, int device);
    ~Engine();

    // A frame between the three phases every registration goes through: Begin* (ingest, motion initialisation, arming
    // the device tail, sampling, the state upload), the ICP launch (solo: LaunchIcp; or a grouped launch shared with
    // other handles, RegisterBatch), FinishFrame (verdict, map update, summary). RegisterFrame / RegisterDevice /
    // RegisterStaged run them back to back. A robust registration (robust_registration) repeats the first two per
    // attempt: EndAttempt decides an attempt and, when it is rejected, begins the next one up to its launch.
    // The grouped ICP launches of RegisterBatch, one per kind of joining frame: solver GN (k_gn_persistent), and solver
    // CERES with the nearest-neighbour strategy, CERES with the distance-based strategy and ROBUST (k_lm_persistent's
    // modes); the attempts of robust registrations in four kinds of their own, the same four solvers.
    enum {
        kJoinsNone = -1, kJoinsGn = 0, kJoinsCeresNearest, kJoinsCeresDistance, kJoinsRobust,
        kJoinsLadderGn, kJoinsLadderCeresNearest, kJoinsLadderCeresDistance, kJoinsLadderRobust, kJoinKinds
    };
    struct PendingFrame {
        size_t n = 0;
        cticp_summary *out = nullptr;
        std::chrono::steady_clock::time_point t_start, t_try;
        double t_initialization = 0, relative_orientation = 0;
        FrameInfo info;
        Summary summary;
        MotionModel caller_model;
        bool default_model = false;   // the handle's default motion model applies (caller_model absent)
        int launches0 = 0;
        cticp_icp_options icp_options{};
        bool ran_icp = false, early_return = false;
        bool icp_pending = false;     // a registration (attempt) waits for its ICP launch and its TryRegisterEnd
        bool icp_launched = false;
        int joins = kJoinsNone;       // the grouped launch its ICP may run in (persistent loop, armed device tail)
        // the robust ladder (RobustRegistrationAttempt): icp_options are the attempt's registration options, summary its
        // summary
        bool ladder = false, ladder_accepted = false;
        int attempt = 0, robust_level = 0;
        double sample_voxel_size = 0;
        HostFrame ladder_initial;
        RobustDecision ladder_decision{};   // of the last decided attempt
    };
    void BeginFrame(const ScanView &scan, uint32_t frame_id, const cticp_frame *initial_estimate, cticp_summary *out,
                    const cticp_motion_prior *motion_model, PendingFrame &f);
    void BeginDevice(ScanView scan, cudaStream_t producer, uint32_t frame_id, const cticp_frame *initial_estimate,
                     cticp_summary *out, const cticp_motion_prior *motion_model, PendingFrame &f);
    void BeginStaged(int64_t slot, uint32_t frame_id, cticp_summary *out, PendingFrame &f);
    // the solo launch when still pending (each remaining attempt of a robust ladder: launch, EndAttempt), then FinishFrame
    void CompleteFrame(PendingFrame &f);
    // the solo ICP launch of the pending registration (attempt), unless a grouped launch ran it
    void LaunchPending(PendingFrame &f);
    // a robust registration after its attempt's ICP launch: the verdict and the decision. Accepted: f.ladder_accepted,
    // ready for CompleteFrame. Rejected: the next attempt is begun and waits for its launch (f.icp_pending, f.joins).
    void EndAttempt(PendingFrame &f);
    // the device tail of the launched attempt (k_frame_policy + the speculative map update), when armed; EndAttempt and
    // TryRegisterEnd enqueue it themselves if nobody did
    void EnqueueTail();
    // a joining frame's registration in a grouped launch (valid until FinishFrame)
    GnProblem IcpProblem(const PendingFrame &f) const;
    // the same for a CERES / ROBUST frame: prepares this handle's LM buffers for it (IcpSolver::PrepareCeres) on the
    // engine's stream, then records IcpReadyEvent again behind that work
    LmProblem CeresProblem(const PendingFrame &f);
    // recorded on the engine's stream after the state upload and the sampling of the pending frame (and CeresProblem)
    cudaEvent_t IcpReadyEvent() const { return ev_[1].get(); }
    // the grouped launch that ran the pending frame's ICP is enqueued, `launched` recorded behind it; `groups` problems
    void AdoptGroupedIcp(PendingFrame &f, cudaEvent_t launched, int groups);
    void FinishFrame(PendingFrame &f);
    // recorded behind a grouped launch this engine's stream carried (RegisterBatch)
    cudaEvent_t GroupDoneEvent() const { return ev_group_done_.get(); }

    void RegisterFrame(const ScanView &scan, uint32_t frame_id, const cticp_frame *initial_estimate, cticp_summary *out,
                       const cticp_motion_prior *motion_model = nullptr);
    // RegisterFrame on a scan in device memory; producer: the stream whose work wrote it (nullptr = legacy default stream)
    void RegisterDevice(ScanView scan, cudaStream_t producer, uint32_t frame_id, const cticp_frame *initial_estimate,
                        cticp_summary *out, const cticp_motion_prior *motion_model);
    // WritePoints into a sink in device memory, enqueued on the engine's stream; `consumer` is made to wait for it
    int64_t WritePointsDevice(int which, const cticp_cloud_sink &sink, cudaStream_t consumer);
    void SetCallback(cticp_event_fn fn, void *user) { callback_ = fn; callback_user_ = user; }
    const cticp_odometry_options &Options() const { return options_; }
    // device-resident input: pack + copy a scan to HBM now, register it later
    int64_t StageFrame(const ScanView &scan);
    int64_t WritePoints(int which, const cticp_cloud_sink &sink);
    void RegisterStaged(int64_t slot, uint32_t frame_id, cticp_summary *out);
    void ClearStaged();
    void TimerStart();
    double TimerStop();
    void FlushL2(size_t bytes);
    int64_t GetPoints(int which, cticp_wpoint *dst, size_t cap);
    // RegistrationSummary's point vectors (odometry.cpp:462-486,597) produced EAGERLY by every RegisterFrame: bit
    // `which` of the mask (CTICP_POINTS_*) selects a vector. 0 (default): computed on demand by GetPoints / WritePoints.
    void SetSummaryPoints(int mask);
    const std::vector<HostFrame> &Trajectory() const { return trajectory_; }
    int64_t MapSize();
    void Reset();
    DeviceMap &Map() { return *map_; }
    IcpSolver &Solver() { return *icp_; }
    cudaStream_t Stream() const { return stream_.get(); }
    int Device() const { return device_; }
    cticp_device_timing LastTiming();   // synchronises on the last frame's final event
    void SetTimeGather(bool on) { icp_->set_time_gather(on); }
    // snapshots (snapshot.cu): Save returns the snapshot's size and, with dst, writes it (cap_bytes below the size is
    // refused); Load builds a handle on `device` from a snapshot (options nullptr: the saved ones); Clone builds one holding
    // the same state on `device`, copied device to device. All three wait for the work queued on the streams.
    int64_t Save(void *dst, size_t cap_bytes);
    static std::unique_ptr<Engine> Load(const void *src, size_t n_bytes, const cticp_odometry_options *options, int device);
    std::unique_ptr<Engine> Clone(int device);
    void EnableSharding(const void *unique_id, int rank, int world);
    void DestroySharding();
    int ShardingMode() const { return shard_world_ <= 1 ? 0 : (icp_ && icp_->peers_ready() ? 2 : 1); }

private:
    void InitializeMotion(const FrameInfo &info, const cticp_frame *initial_estimate);
    void DrainStreams();
    snap::HostState SnapshotHostState() const;
    void RestoreHostState(const snap::HostState &s, std::vector<HostFrame> trajectory);
    void ResolvePoints(int which, const float4 **out_pts, const float4 **out_lo, const double **out_world, size_t *out_count);
    // The owning members below are released in reverse declaration order once the destructor has synchronised stream_:
    // stream_ comes first so that it is destroyed after everything that was enqueued on it, the egress stream after its
    // events and buffers.
    cticp::Stream stream_;
    Event ev_producer_, ev_device_egress_;   // device input / output: the caller's stream order
    void IngestImpl(const ScanView &scan,
                    const FrameInfo &info, int64_t staged_slot);
    bool PackScan(const ScanView &scan, double bts, double ets, float4 *dst);
    void PackLoPlane(const ScanView &scan, double bts, double ets, float4 *dst_lo);
    // one parallel region: timestamp min/max → team barrier → (x, y, z, alpha) packing in rounds, the H2D copy of a
    // round enqueued as soon as the round is complete (the copy engine runs while the later rounds are still packed)
    void PackAndUpload(const ScanView &scan, const double *pose_timestamps, double *mn_out, double *mx_out);
    void MinMaxTimestamps(const ScanView &scan, double *mn_out, double *mx_out);
    std::unique_ptr<HostPool> pool_;
    static int HostTeamSize(int ranks_on_node);
    void PrepareFrame(const ScanView &scan, uint32_t frame_id, const cticp_frame *initial_estimate, int64_t staged_slot,
                      cticp_summary *out, const cticp_motion_prior *motion_model, PendingFrame &f);
    const MotionModel *ModelOf(const PendingFrame &f) const;
    void FireEvent(int event, const Summary &rs, const FrameInfo &info);
    cticp_event_fn callback_ = nullptr;
    void *callback_user_ = nullptr;
    bool frame_world_valid_ = false;
    bool fused_map_update_ = true;     // CTICP_FUSED_MAP_UPDATE=0: transform / evict / insert as separate launches
    bool fused_sampling_ = true;       // CTICP_FUSED_SAMPLING=0: the two grid selections as separate launches
    bool keypoints_sampled_ = false;   // the keypoints of the coming first attempt were sampled with the frame   // d_frame_world holds the sub-sampled frame under last_frame_
    struct StagedScan {
        DeviceArray<float4> d_points;
        DeviceArray<float4> d_lo;   // residual plane, float64 scans only (se3.cuh load_raw)
        size_t n = 0;
        double t_min = 0, t_max = 0;
    };
    std::vector<StagedScan> staged_;
    Event timer_ev_[2];
    DeviceArray<unsigned char> d_flush_;
    void TryRegisterBegin(const FrameInfo &info, cticp_icp_options &options, Summary &rs, double sample_voxel_size,
                          const MotionModel *mm, int attempt_idx);
    void LaunchIcp(const cticp_icp_options &options);
    void TryRegisterEnd(const FrameInfo &info, const cticp_icp_options &options, Summary &rs);
    bool verdict_by_icp_kernel_ = false;   // the last ICP launch decided the frame's tail itself (CTICP_TAIL_IN_KERNEL)
    bool AssessRegistration(Summary &s) const;
    // the robust ladder (RobustRegistration) in steps: engine.cu
    void BeginLadder(PendingFrame &f);
    void BeginAttempt(PendingFrame &f);
    void IncreaseRobustness(PendingFrame &f);
    RobustPolicyIn LadderInputs(const PendingFrame &f) const;
    double LadderSampleSize(int k, int level) const;
    bool ladder_tail_ = false;   // the current robust frame's attempts take the device tail
    void ArmTail(double relative_orientation);
    int JoinKind(const cticp_icp_options &o);
    void ComputeSummaryMetrics(Summary &s, int k);
    void UpdateMap(Summary &s, int registered_fid, const RobustDecision *robust);
    // The tail of a plain registration decided on the device (frame_policy.h): TryRegister enqueues k_frame_policy and a
    // speculative k_map_update_fused right behind the ICP kernel, then waits for the verdict in mapped pinned memory — no
    // copy-engine operation and no host round trip between the ICP loop and the map update.
    bool device_tail_ = true;      // CTICP_DEVICE_TAIL=0: AssessRegistration / UpdateMap on the host for every frame
    bool tail_in_kernel_ = false;  // CTICP_TAIL_IN_KERNEL=1: solver GN's persistent kernel decides the tail itself at the end of
                                   // its loop instead of a separate k_frame_policy launch (three launches per frame; the
                                   // default keeps the policy in its own one-warp kernel, the same for every solver)
    bool tail_armed_ = false;      // the coming TryRegister enqueues the device tail (tail_in_ is filled)
    bool tail_launched_ = false;   // the last TryRegister did: h_verdict_ holds this frame's verdict
    FramePolicyIn tail_in_{};
    RobustPolicyIn tail_robust_{};   // the robust ladder's inputs of the coming attempt (enabled = 0 on the plain path)
    DeviceArray<FrameVerdict> d_verdict_;
    PinnedArray<FrameVerdict> h_verdict_{cudaHostAllocMapped};
    FrameVerdict *h_verdict_dev_ = nullptr;   // its device address
    unsigned verdict_seq_ = 0;
    int tail_launches_ = 0;
    void WaitVerdict(unsigned seq);
    void AdoptDeviceMapUpdate(Summary &s);
    // the registration state goes up on a second stream while the sampler runs (the ICP kernel waits for its event)
    cticp::Stream aux_stream_;
    Event ev_state_up_;
    Event ev_group_done_;
    void FillSummary(const Summary &s, cticp_summary *out) const;
    // grid-size hint for the ICP kernels: the keypoint count is only known on the device when they are enqueued, so
    // the host sizes the grid from the previous registration (keypoint counts change slowly) with 25% head-room;
    // the kernels stay correct for any count (warps loop)
    size_t KeypointHint() const {
        return last_num_keypoints_ ? std::min(pipe_->n(), last_num_keypoints_ + last_num_keypoints_ / 4 + 64) : pipe_->n();
    }
    size_t last_num_keypoints_ = 0;
    // the previous frame's sub-sampled point count F, which sizes the device tail's head-room (ArmTail): h_counts()[1],
    // or, on a handle loaded or cloned from a snapshot until its first frame finishes, the saved handle's value (the
    // pipeline's counts stay those of a fresh handle, so get_points answers as on one)
    int PrevFramePoints() const {
        return restored_prev_frame_points_ >= 0 ? restored_prev_frame_points_ : std::max(0, pipe_->h_counts()[1]);
    }
    int restored_prev_frame_points_ = -1;
    bool frame_events_recorded_ = false;   // ev_[0..3] hold a frame's events (LastTiming may query them)
    bool keypoints_in_summary_ = false;   // the last TryRegister's ICP succeeded: RegistrationSummary::keypoints is filled
    static uint64_t ShuffleCounter(int registered_fid, int purpose) {
        return (uint64_t(uint32_t(registered_fid)) << 8) | uint64_t(purpose & 0xff);
    }

    cticp_odometry_options options_;
    int device_;
    std::unique_ptr<DeviceMap> map_;
    std::unique_ptr<FramePipeline> pipe_;
    std::unique_ptr<IcpSolver> icp_;
    DeviceArray<IcpState> d_state_;
    PinnedArray<IcpState> h_state_;
    std::vector<HostFrame> trajectory_;
    MotionModel default_motion_model_;
    int registered_frames_ = 0;
    int robust_num_consecutive_failures_ = 0;
    bool suspect_registration_error_ = false;
    int next_robust_level_ = 0;
    struct {
        double cum_distance = 0, cum_orientation = 0;
        int skipped_frames = 0, total_insertions = 0;
    } tracker_;
    // state of the last registered frame (for GetPoints)
    HostFrame last_frame_;
    FrameInfo last_info_;
    bool last_all_world_valid_ = false, last_kp_world_valid_ = false;
    DeviceArray<double> d_kp_world_;
    // eager egress of the summary vectors: world coordinates (+ source indices) to pinned host memory on a second
    // stream, overlapped with the map update; GetPoints assembles the 64-byte records on the host team
    void EnqueueEgress(const HostFrame &f, bool ran_icp);
    void AllocEgress();
    int summary_points_mask_ = 0;
    cticp::Stream egress_stream_;
    Event ev_egress_main_, ev_egress_done_;
    static constexpr int kEgressChunks = 4;   // the N world points go back in pieces: the host assembles the
    Event ev_egress_chunk_[kEgressChunks];    // records of piece i while piece i + 1 is still on the bus
    bool egress_pending_ = false;           // ev_egress_done_ recorded, next frame's upload must wait for it
    bool egress_valid_[3] = {false, false, false};
    size_t egress_count_[3] = {0, 0, 0};
    PinnedArray<double> h_world_[3];     // corrected / all corrected / keypoints, xyz triples
    PinnedArray<uint32_t> h_src_[3];     // index into the scan (corrected, keypoints)
    bool scan_in_staging_ = false;          // the pinned staging buffer holds the last registered scan
    // timing
    cticp_device_timing timing_{};
    Event ev_[6];
    bool tail_event_valid_ = false;    // ev_[3] (end of the last frame's map update) has been recorded and not yet waited on
    bool staging_in_flight_ = false;   // the pinned staging buffer may still feed an H2D copy
    // multi-GPU
    void *nccl_comm_ = nullptr;
    int shard_rank_ = 0, shard_world_ = 1;
    // NVLink peer mailboxes of the in-kernel exchange (peer_exchange.cuh, nccl_shard.cu)
    bool ConnectPeers();
    void DisconnectPeers();
    void *d_mailbox_ = nullptr;
    std::vector<void *> peer_mapped_;
};

// One frame of RegisterBatch (odometry_batch.cu): the arguments of the single-frame entry `kind` (CTICP_BATCH_*) names
struct BatchItem {
    Engine *engine = nullptr;
    int kind = CTICP_BATCH_HOST;
    ScanView scan;                 // HOST, DEVICE (scan.n: the staged slot's size is looked up by the engine)
    cudaStream_t producer = nullptr;
    int64_t slot = -1;
    uint32_t frame_id = 0;
    const cticp_frame *initial_estimate = nullptr;
    const cticp_motion_prior *motion_model = nullptr;
    cticp_summary *out = nullptr;
    std::exception_ptr error;      // out: what the item's single-frame call would have thrown
};
// One frame on each engine (all distinct, one device, none sharded), the eligible ICP loops in one grouped launch per
// kind, PendingFrame::joins (cticp_odometry_register_batch has the contract). A failing item ends alone with its exception in `error`.
void RegisterBatch(std::vector<BatchItem> &items);

// standalone maps (snapshot.cu): the size of the map snapshot and, with dst, the snapshot; a map snapshot's validation
int64_t SaveMap(DeviceMap &map, void *dst, size_t cap_bytes);
void ValidateMapSnapshot(const void *src, size_t n_bytes, snap::Parsed *p);

// conversions shared with capi.cu
HostPose PoseFromC(const cticp_pose &c);
cticp_pose PoseToC(const HostPose &p);
HostFrame FrameFromC(const cticp_frame &c);
cticp_frame FrameToC(const HostFrame &f);

}  // namespace cticp
