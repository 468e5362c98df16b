// icp.h — device-side state and host-side driver of the registration solvers (GN now; CERES-as-LM in icp_lm.cu).
#pragma once
#include <cuda_runtime.h>

#include <vector>

#include "../../include/cticp.h"
#include "device_map.h"

namespace cticp {

constexpr int kAcc = 96;            // accumulator width: 78 (A upper) + 12 (b) + 6 stats
constexpr int kAccUsed = 90;        // n keypoints used
constexpr int kAccSumSq = 91;       // Σ scalar²
constexpr int kAccStencil = 92;     // Σ map points inside the stencils
constexpr int kAccKeypoints = 93;   // keypoints visited
constexpr int kAccValidNb = 94;     // keypoints with >= min neighbors

// Everything one ICP needs across iterations lives on the device so that all iterations can be enqueued without a
// host round trip (the reference's loop, src/ct_icp/ct_icp.cpp:745-981, is sequential on the host).
struct IcpState {
    double qb[4], tb[3], qe[4], te[3];     // pose pair being optimised (quat x,y,z,w)
    double prev_tb[3], prev_te[3];         // PreviousFrameMotionModel state (previous frame begin / end translation)
    double prev_qe[4];
    double beta_location, beta_cv, beta_small, beta_orientation;
    int has_motion_model;
    int iter;            // iterations executed
    int done;            // convergence or failure: later launches become no-ops
    int failed;          // "not enough keypoints" (ct_icp.cpp:860-871)
    int n_used;          // residuals of the last linearisation
    int n_keypoints;     // keypoints visited in the last iteration
    double x_norm;       // ‖x‖ of the last GN step
    // slerp constants of the current pose pair (se3.cuh SlerpConsts), refreshed by every pose update
    double slerp_theta, slerp_inv_sin;
    int slerp_linear, slerp_negate;
    unsigned long long stat_keypoint_iters, stat_stencil_points;
    unsigned long long dbg_t[4];   // SM cycle stamps of the last iteration (CTICP_DEBUG_TIMERS builds)
    // SM cycles of the solver CTA over the persistent GN loop: whole loop, and the reduce + solve part of it (the rest is
    // the neighborhood / residual assembly it waits for) — the split behind ICPSummary::avg_duration_neighborhood / _solve
    unsigned long long cycles_total, cycles_solve;
};

inline void icp_state_refresh_slerp(IcpState &S) {
    const SlerpConsts c = slerp_consts(Q4{S.qb[0], S.qb[1], S.qb[2], S.qb[3]}, Q4{S.qe[0], S.qe[1], S.qe[2], S.qe[3]});
    S.slerp_theta = c.theta;
    S.slerp_inv_sin = c.inv_sin;
    S.slerp_linear = c.linear;
    S.slerp_negate = c.negate;
}

// Host-side description of the peer mailboxes (mirrors PeerLinks of peer_exchange.cuh without device code)
constexpr int kMaxPeerRanks = 8;
struct PeerLinksHost {
    int world = 1, rank = 0;
    unsigned long long *inbox[kMaxPeerRanks] = {};
    unsigned int *seq = nullptr;
    long long timeout_cycles = 0;   // 0 = the default of peer_exchange.cuh
};

// -DCTICP_DEBUG_TIMERS builds (tools/ab_variants.sh "timers"): clock64 stamps of the solver CTAs, printed by the host when
// the environment has CTICP_DEBUG_TIMERS. (%globaltimer proved far too slow to read: it tripled the kernel time; only
// differences taken on the same SM are meaningful.)
#ifdef CTICP_DEBUG_TIMERS
#define CT_STAMP(...) __VA_ARGS__
#else
#define CT_STAMP(...)
#endif

struct GnParams {
    int r;                      // stencil radius (voxels)
    int level;                  // map level searched
    double radius;              // search radius (default_radius)
    int kmax, kmin;             // max / min_number_neighbors
    double max_dist_to_plane;   // max_dist_to_plane_ct_icp
    double threshold_norm;      // threshold_orientation_norm (GN stop criterion on ‖x‖, ct_icp.cpp:978)
    int shard_rank, shard_world;   // keypoint sharding (multi-GPU); 0/1 when single
    int debug_flags;               // profiling only (env CTICP_DEBUG_FLAGS): 1 = skip the solve, 2 = skip the gather work,
                                   // 8 = no paired tile schedule in k_gn_persistent (bit-identity tests)
    double bucket_scale;           // 32 / radius^2: d2 → histogram bucket of the k-nearest selection (gather_select.cuh)
    const float4 *kp_lo;           // residual plane of the keypoints (nullptr: float32-representable; load_raw, se3.cuh)
    unsigned long long *dbg_warp;  // -DCTICP_DEBUG_TIMERS builds with CTICP_DEBUG_TIMERS set: per-warp phase stamps (icp_gn.cu)
    int rigid_first;               // motion compensation NONE / CONSTANT_VELOCITY: the keypoints enter the first iteration
                                   // transformed by the END pose alone (TransformPoint, odometry.cpp:171-184), afterwards GN
                                   // interpolates like always (ct_icp.cpp:964-966)
};

// bound of every wait of the persistent loops on another CTA (k_gn_persistent's hand-off, k_lm_persistent's group barrier)
constexpr long long kLoopSyncTimeout = 4000000000LL;   // SM cycles (~2 s)

// CTAs of the persistent kernels (icp_batch.cu): GatherBlocks is the worker / gather CTA count of a solo launch for
// k_hint keypoints; BatchGatherCtas deals the co-resident CTAs of a batched launch over its problems (contract there).
int GatherBlocks(size_t k_hint, int max_blocks, int kp_per_cta);
void BatchGatherCtas(const size_t *n, int batch, int coresident, int kp_per_cta, int *gather);

struct FrameTailArgs;   // frame_policy.h
struct LmState;            // icp_lm.cu
struct DistanceStrategy;   // icp_lm.cu
struct ResidualBlock;      // lm_functor.cuh

// One registration of a grouped Gauss-Newton launch (IcpSolver::EnqueueGaussNewtonGroups)
struct GnProblem {
    const DeviceMap *map;
    const cticp_icp_options *opt;
    const float4 *keypoints;
    const float4 *keypoints_lo;     // residual plane of the keypoints (nullptr: none; se3.cuh load_raw)
    const int *d_num_keypoints;     // device keypoint count; nullptr: exactly n keypoints
    size_t n;                       // the keypoint count, or with d_num_keypoints the estimate a solo launch sizes its grid
                                    // from (EnqueueGaussNewton's k_upper)
    int num_iters;
    IcpState *d_state;
};

// One registration of a grouped CERES / ROBUST launch (IcpSolver::EnqueueCeresGroups). Options checked by CheckCeresOptions;
// the per-keypoint buffers and the uploaded strategy as IcpSolver::PrepareCeres leaves them.
struct LmProblem {
    const DeviceMap *map;
    const cticp_icp_options *opt;
    const cticp_strategy_options *strategy;
    const float4 *keypoints;
    const float4 *keypoints_lo;     // residual plane of the keypoints (nullptr: none; se3.cuh load_raw)
    const int *d_num_keypoints;     // device keypoint count; nullptr: exactly n keypoints
    size_t n;                       // the keypoint count, or with d_num_keypoints the estimate a solo launch sizes its grid
                                    // from (EnqueueCeres's k_hint)
    IcpState *d_state;
    ResidualBlock *blocks;          // ncn residual blocks per keypoint
    int *sel_idx;                   // ncn per keypoint
    unsigned char *classes;         // solver ROBUST: one per keypoint, NEIGHBORHOOD_TYPE::NONE on entry
    const DistanceStrategy *distance;   // CERES with the distance-based strategy: its parameters and the map's levels
};

class IcpSolver {
public:
    explicit IcpSolver(cudaStream_t stream);

    // d_keypoints: float4 (raw xyz fp32, alpha fp32); d_num_keypoints: device int; upper bound for grid sizing.
    // Enqueues `num_iters` GN iterations on the stream; state is read back by the caller.
    // tail != nullptr: the frame's tail (frame_policy.h) is decided by the kernel that ends the loop when that is the
    // persistent one — returns true then (the verdict is written by k_gn_persistent's solver CTA); false: the caller
    // launches k_frame_policy itself.
    bool EnqueueGaussNewton(const DeviceMap &map, const cticp_icp_options &opt, const float4 *d_keypoints,
                            const int *d_num_keypoints, size_t k_upper, int num_iters, IcpState *d_state,
                            int shard_rank = 0, int shard_world = 1, void *nccl_comm = nullptr,
                            const FrameTailArgs *tail = nullptr);

    // B independent Gauss-Newton registrations against `map` with shared options, in ONE launch of the persistent kernel
    // (EnqueueGaussNewtonGroups, every group on the same map). Problem b's h_n[b] keypoints are at
    // [kp_base_b, kp_base_b + h_n[b]) of d_keypoints, kp_base_b = h_n[0] + … + h_n[b - 1] (the residual plane, when
    // set_keypoints_lo gave one, alike); its state is d_states[b].
    void EnqueueGaussNewtonBatch(const DeviceMap &map, const cticp_icp_options &opt, int batch, const size_t *h_n,
                                 const float4 *d_keypoints, int num_iters, IcpState *d_states);
    // B independent Gauss-Newton registrations, each with its own map, options, keypoints and iteration count, in ONE
    // launch of the grouped persistent kernel (k_gn_persistent<false, true>) on this solver's stream, with this solver's
    // loop words and group table. CTA policy and its bit-identity contract with the solo launch: BatchGatherCtas
    // (icp_batch.cu) on the problems' n. Throws CapacityError when the device cannot hold two CTAs per problem;
    // requires batch_supported(). The table is built on the host before this returns: `problems` may go afterwards.
    void EnqueueGaussNewtonGroups(const GnProblem *problems, int batch);
    // the batch has no launch-per-iteration form (CTICP_PERSISTENT=0) and cannot use grid-wide barriers, which would
    // couple groups with different iteration counts (-DCTICP_GN_GRID_BARRIERS builds)
    bool batch_supported() const;

    // solver CERES reproduced as a device Levenberg-Marquardt / IRLS loop (icp_lm.cu)
    // k_hint sizes the grids (estimate of the keypoint count), k_capacity the per-keypoint buffers (upper bound)
    void EnqueueCeres(const DeviceMap &map, const cticp_icp_options &opt, const cticp_strategy_options &strategy,
                      const float4 *d_keypoints, const int *d_num_keypoints, size_t k_hint, size_t k_capacity,
                      IcpState *d_state, int shard_rank = 0, int shard_world = 1, void *nccl_comm = nullptr);
    // the option checks of EnqueueCeres, without touching the device: UnsupportedError / std::invalid_argument
    void CheckCeresOptions(const DeviceMap &map, const cticp_icp_options &opt, const cticp_strategy_options &strategy) const;
    // B independent CERES / ROBUST registrations against `map` with shared options and strategy, in ONE launch of the
    // persistent LM kernel (EnqueueCeresGroups, every group on the same map, this solver's buffers). Keypoints and states
    // are laid out as for EnqueueGaussNewtonBatch.
    void EnqueueCeresBatch(const DeviceMap &map, const cticp_icp_options &opt, const cticp_strategy_options &strategy,
                           int batch, const size_t *h_n, const float4 *d_keypoints, IcpState *d_states);
    // What EnqueueCeres does before its launch, for a registration that a grouped launch will run: the option checks, this
    // solver's per-keypoint buffers sized for k_capacity keypoints, the strategy upload and ROBUST's class reset, all on
    // this solver's stream. Returns the problem with this solver's buffers and residual plane (set_keypoints_lo).
    LmProblem PrepareCeres(const DeviceMap &map, const cticp_icp_options &opt, const cticp_strategy_options &strategy,
                           const float4 *d_keypoints, const int *d_num_keypoints, size_t k_hint, size_t k_capacity,
                           IcpState *d_state);
    // B independent CERES / ROBUST registrations of one k_lm_persistent mode (CERES nearest neighbour, CERES
    // distance-based, ROBUST), each with its own map, options, keypoints, state and buffers, in ONE launch of the grouped
    // persistent LM kernel (groups separated by group barriers) on this solver's stream, with this solver's group area and
    // table; one problem takes the solo launch. CTA policy and its bit-identity contract with the solo launch:
    // BatchGatherCtas (icp_batch.cu) on the problems' n with the LM kernel's co-resident count. A group whose barrier
    // times out ends with failed = 2 without holding up the others. Throws CapacityError when the device cannot hold two
    // CTAs per problem; requires use_persistent(). The table is built on the host before this returns.
    void EnqueueCeresGroups(const LmProblem *problems, int batch);
    bool use_persistent() const { return use_persistent_; }

    // single linearisation at the current state → A (12x12, after 1/n and regularisers), b, n_used (debug tap)
    void NormalEquations(const DeviceMap &map, const cticp_icp_options &opt, const float4 *d_keypoints,
                         const int *d_num_keypoints, size_t k_upper, IcpState *d_state, double *h_A144, double *h_b12,
                         int *h_n_used);

    // neighbor lists for queries (fp64 xyz on device): out_points n*kmax*3 (farthest first), out_counts n
    void Neighborhoods(const DeviceMap &map, const double *d_queries, size_t n, int kmax, double *d_out_points,
                       int *d_out_counts);
    void RadiusSearch(const DeviceMap &map, const double *d_queries, const double *d_radiuses, size_t n, int kmax,
                      const double *sensor_location, double *d_out_points, int *d_out_counts);

    // residual plane of the keypoint array the next Enqueue*/NormalEquations calls are given (nullptr: none; se3.cuh load_raw)
    void set_keypoints_lo(const float4 *d_lo) { kp_lo_ = d_lo; }
    int launches() const { return launches_; }
    float gather_ms() const { return gather_ms_; }
    void reset_timing() { gather_ms_ = 0.f; gather_launches_ = 0; }
    int gather_launches() const { return gather_launches_; }
    void set_time_gather(bool on) { time_gather_ = on; }
    void set_persistent(bool on) { use_persistent_ = on; }
    // -DCTICP_DEBUG_TIMERS builds: per-warp cycles of the gather phases (A pose + voxel, B gather + selection, C epilogue, D rows)
    // of the last persistent GN loop, mean / p90 / max over the warps per iteration, on stderr
    void PrintWarpStamps(int iters);
    void CollectGatherTiming();   // after a stream sync: accumulates the event pairs recorded since the last call
    // multi-GPU: d_acc_[0..kAcc) ← Σ over ranks of d_acc_, in place: over the NVLink peer mailboxes when they are
    // connected (k_peer_allreduce, peer_exchange.cuh), else ncclAllReduce (nccl_shard.cu). d_state receives the
    // failure flag if a peer never answers.
    void AllReduceAccumulator(void *nccl_comm, IcpState *d_state);
    // peer mailboxes (nccl_shard.cu sets them up); world == 1 disconnects
    void SetPeerLinks(const PeerLinksHost &links);
    // loads the modules of the sharded kernels now (lazy loading would otherwise hit the first sharded frame of one rank
    // while its peers already wait in the exchange)
    void PreloadShardedKernels();
    void PreloadLmKernels();   // icp_lm.cu
    void NcclAllReduceAccumulator(void *nccl_comm);   // nccl_shard.cu
    double *acc_buffer() const { return d_acc_.data(); }
    bool peers_ready() const { return peers_ready_; }

private:
    void EnsurePartials(int blocks);
    void EnsureLmBuffers(size_t k_upper);
    void DebugLmTrace(void *d_lm);
    int lm_coresident_[9] = {};   // k_lm_persistent<mode, peers> at mode * 2 + peers, <mode, false, true> at 6 + mode
    GnParams MakeParams(const DeviceMap &map, const cticp_icp_options &opt) const;
    int GnCoresident(bool peers);          // co-resident CTAs of k_gn_persistent<peers> on this device
    unsigned int ReserveLoopTags(int rows, int groups, int num_iters);   // k_gn_persistent's words and tags (icp_gn.cu)
    // co-resident CTAs of a k_lm_persistent instantiation with `smem` bytes of dynamic shared memory (icp_lm.cu)
    int LmCoresident(int variant, void *kernel, size_t smem);
    bool UploadLmStrategy(const DeviceMap &map, const cticp_icp_options &opt, const cticp_strategy_options &strategy);

    cudaStream_t stream_;
    const float4 *kp_lo_ = nullptr;
    DeviceArray<double> d_partials_;   // kAcc per CTA (grow-only)
    DeviceArray<unsigned long long> d_dbg_warp_;   // [kDbgIters][warps][kDbgSlots]
    int dbg_warps_ = 0;
    DeviceArray<double> d_sys_;      // 12*12 + 12 + 4 debug output of the solve kernel
    DeviceArray<double> d_acc_;      // reduced accumulator (multi-GPU all-reduce buffer)
    DeviceArray<unsigned int> d_ticket_;   // last-CTA-done counter of k_gn_iterate
    DeviceArray<unsigned long long> d_loop_rows_;   // k_gn_persistent: tagged partial rows of the gather CTAs (grow-only)
    DeviceArray<unsigned long long> d_loop_pose_;   // k_gn_persistent: tagged pose words, one block per group (grow-only)
    unsigned int loop_tag_ = 1;                     // next tag to hand out (never 0)
    DeviceArray<unsigned char> d_gn_table_;    // grouped GN launches: GnGroup table | first_cta | counts (grow-only)
    std::vector<unsigned char> h_gn_table_;
    DeviceArray<unsigned char> d_lm_table_;    // grouped LM launches: LmGroup table | first_cta | counts (grow-only)
    std::vector<unsigned char> h_lm_table_;
    // solver CERES (icp_lm.cu)
    DeviceArray<LmState> d_lm_state_;
    DeviceArray<unsigned long long> d_lm_stats_;
    DeviceArray<ResidualBlock> d_lm_blocks_;
    DeviceArray<int> d_lm_sel_;
    DeviceArray<unsigned char> d_lm_classes_;   // solver ROBUST: slam::NEIGHBORHOOD_TYPE per keypoint
    DeviceArray<DistanceStrategy> d_lm_strategy_;  // DistanceBasedStrategy parameters + every map level
    DeviceArray<char> d_lm_groups_;             // batched launches: per group an LmState, a stats line and the barrier words (grow-only)
    int launches_ = 0;
    float gather_ms_ = 0.f;
    int gather_launches_ = 0;
    bool time_gather_ = false;
    static constexpr int kMaxEvents = 64;
    Event ev_begin_[kMaxEvents], ev_end_[kMaxEvents];
    int ev_used_ = 0;
    int num_sms_ = 132;
    int max_coresident_[2] = {0, 0};   // k_gn_persistent<false / true>
    int kp_per_cta_ = 8;               // keypoints per gather CTA below which the persistent grid is not widened further
    bool use_persistent_ = true;
    PeerLinksHost links_host_;
    bool peers_ready_ = false;
};

}  // namespace cticp
