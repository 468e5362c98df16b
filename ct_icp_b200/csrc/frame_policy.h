// frame_policy.h — the tail of RegisterFrame decided on the device.
//
// The reference decides on the host, after the ICP, whether the registration is acceptable (AssessRegistration,
// src/ct_icp/odometry.cpp:604-684) and whether the frame is inserted into the map (UpdateMap, :855-953). Every input of
// those decisions is either on the device when the ICP loop ends (the pose pair, the failure flag, the frame's point count)
// or known to the host before the loop starts (thresholds, the insertion tracker, the previous pose). So the engine
// enqueues, right behind the ICP kernel and without waiting for it:
//
//     k_frame_policy      one warp: evaluates the decision, writes a FrameVerdict to device memory AND to mapped pinned host
//                         memory (state + counters + decision + sequence number: the only thing the host waits for)
//     k_map_update_fused  reads the pose pair and the decision from the device copy of the verdict
//
// and then spins on the sequence number. One stream, no copy-engine operation and no host round trip between the ICP loop
// and the map update; the host learns the poses while the map update is already running.
//
// Covers the plain registration path and every attempt of the robust ladder (robust_registration = 1, decided by
// robust_attempt_decide below), under no callbacks, motion compensation CONTINUOUS and the fused map update; every other
// configuration keeps the host-side tail (engine.cu UpdateMap).
#pragma once
#include <cstddef>

#include "icp.h"
#include "se3.cuh"

namespace cticp {

enum FrameAction : int {
    kFrameSkip = 0,       // no map update (quit_on_error after a failed assessment, or an ICP error the host turns into an exception)
    kFrameEvict = 1,      // transform + RemoveElementsFarFromLocation, no insertion
    kFrameInsert = 2,     // transform + eviction + InsertPointCloud
    kFrameDeferred = 3,   // nothing done: the frame has more points than the tables were prepared for — the host runs UpdateMap
    kFrameRetry = 4,      // robust ladder: the attempt is rejected and another one follows — no map update
};

struct FramePolicyIn {   // host → k_frame_policy (kernel parameter)
    double distance_error_threshold, orientation_error_threshold;
    double relative_orientation;   // previous end pose vs the INITIAL estimate's end pose (odometry.cpp:429-431): host-known
    double insertion_ego_rotation_threshold;
    int quit_on_error;
    int has_insertions;            // tracker: total_insertions > 0
    int skipped_enough;            // tracker: skipped_frames > insertion_threshold_frames_skipped
    int do_no_insert, always_insert;
    int room_for;                  // the map tables have room for this many new points (DeviceMap::EnsureRoomFor)
    unsigned seq;
};

struct FrameVerdict {
    IcpState state;          // final registration state (what the D2H copy of d_state_ used to bring back)
    int counts[4];           // N, F, K of the frame (FramePipeline counters)
    int assess_ok;           // AssessRegistration
    int add_points_policy;   // UpdateMap's decision before the do_no_insert / always_insert overrides (summary.points_added)
    int action;              // FrameAction
    int next_robust_level;   // robust ladder, accepted attempt: UpdateMap's next_robust_level_ (0 on the plain path)
    double ego_orientation, relative_distance;
    SlerpConsts sc;          // of the final pose pair
    unsigned seq;            // written last (host copy: after a system-wide fence)
    unsigned pad1;
};

// What a kernel that ends a registration is given to decide the frame's tail itself (k_gn_persistent: its solver CTA holds
// the final state in shared memory and writes the verdict before the kernel ends — no k_frame_policy launch, and the host
// sees the poses one kernel boundary earlier)
struct FrameTailArgs {
    FramePolicyIn in;
    const int *counts;    // FramePipeline counters (N, F, K, -)
    FrameVerdict *dv;     // device copy
    FrameVerdict *hv;     // mapped pinned host copy (device address)
    int enabled;
};

// ---- the robust ladder (robust_registration = 1) --------------------------------------------------------------------
// One attempt of RobustRegistration (odometry.cpp:780-852) is decided from its final pose pair and ICP failure flag plus
// what the host knows before the attempt starts. The host tail (engine.cu) and k_frame_policy evaluate the same function.
struct RobustPolicyIn {   // host → k_frame_policy (second kernel parameter; FramePolicyIn holds the shared thresholds)
    double prev_qe[4], prev_te[3];           // trajectory_[k-1].end_pose
    double threshold_relative_orientation;   // robust_threshold_relative_orientation
    double threshold_ego_orientation;        // robust_threshold_ego_orientation
    double relative_trans_threshold;         // robust_relative_trans_threshold
    int num_attempts_when_rotation;          // robust_num_attempts_when_rotation
    int minimal_level;                       // robust_minimal_level
    int number_of_attempts;                  // summary.number_of_attempts once this attempt is counted
    int last_attempt;                        // number_of_attempts >= robust_num_attempts: accepted whatever its assessment
                                             // (= UpdateMap's suspect_registration_error_ if it ends the ladder)
    int consecutive_failures;                // robust_num_consecutive_failures_ after the frame, if this attempt ends it
    int enabled;
};

struct RobustDecision {
    double distance_correction, relative_orientation, ego_orientation, relative_distance;   // of the attempt (:802-821)
    int assess_ok;           // AssessRegistration with the robust branch (:604-684)
    int reject_reason;       // kRejectNone / kRejectError / kRejectRotation / kRejectTranslation (the error message)
    int accepted;            // the ladder ends with this attempt (:823-845)
    int add_points_policy;   // UpdateMap's add_points before do_no_insert / always_insert (summary.points_added)
    int add_points;          // … after them
    int next_robust_level;   // next_robust_level_ after the frame (:890-901)
    int action;              // FrameAction: kFrameRetry for a rejected attempt
};
enum { kRejectNone = 0, kRejectError = 1, kRejectRotation = 2, kRejectTranslation = 3 };

// AssessRegistration with the robust branch, the acceptance rule of RobustRegistration, the robust branch of UpdateMap and
// the insert overrides. `in` supplies distance / orientation_error_threshold, do_no_insert, always_insert and room_for;
// its plain-path fields (relative_orientation, quit_on_error, the tracker) do not apply here. A robust frame never returns
// early on quit_on_error (DoRegister :419-420 skips that branch), so an accepted attempt always updates the map.
CT_HD RobustDecision robust_attempt_decide(const Q4 &qb, const V3 &tb, const Q4 &qe, const V3 &te, int failed,
                                           int frame_points, const FramePolicyIn &in, const RobustPolicyIn &r) {
    RobustDecision d;
    const Q4 prev_q{r.prev_qe[0], r.prev_qe[1], r.prev_qe[2], r.prev_qe[3]};
    const V3 prev_t{r.prev_te[0], r.prev_te[1], r.prev_te[2]};
    d.distance_correction = norm(tb - prev_t);
    d.relative_orientation = angular_distance_deg(prev_q, qe);
    d.ego_orientation = angular_distance_deg(qb, qe);
    d.relative_distance = norm(te - tb);
    const bool large_rotation = d.relative_orientation > r.threshold_relative_orientation ||
                                d.ego_orientation > r.threshold_ego_orientation;
    // AssessRegistration. The reference never copies the attempt's level into summary.robust_level, so the rotation
    // rule always sees level 0 (orc_odometry.h keeps the same quirk)
    int reason = kRejectNone;
    if (d.relative_distance > in.distance_error_threshold) reason = kRejectError;
    else if (d.relative_orientation > in.orientation_error_threshold || d.ego_orientation > in.orientation_error_threshold)
        reason = kRejectError;
    else if (large_rotation && 0 < r.num_attempts_when_rotation) reason = kRejectRotation;
    else if (d.relative_distance > r.relative_trans_threshold) reason = kRejectTranslation;
    d.reject_reason = reason;
    d.assess_ok = (reason == kRejectNone && !failed) ? 1 : 0;
    d.accepted = (d.assess_ok || r.last_attempt) ? 1 : 0;
    // UpdateMap, the robust branch (summary.success is the ICP's: the ladder does not fold the assessment into it)
    bool add = !large_rotation;
    if (r.last_attempt) add = add || (r.consecutive_failures > 5);
    int next = add ? r.minimal_level : r.minimal_level + 1;
    if (failed) next = r.minimal_level + 2;
    else {
        if (large_rotation) next = r.minimal_level + 1;
        if (r.number_of_attempts > 1) next = r.minimal_level + 1;
    }
    d.add_points_policy = add ? 1 : 0;
    d.next_robust_level = next;
    if (in.do_no_insert) add = false;
    if (in.always_insert) add = true;
    d.add_points = add ? 1 : 0;
    int action;
    if (failed == 2 || failed == 3) action = kFrameSkip;   // the host raises an exception
    else if (!d.accepted) action = kFrameRetry;
    else if (add && frame_points > in.room_for) action = kFrameDeferred;
    else action = add ? kFrameInsert : kFrameEvict;
    d.action = action;
    return d;
}

#ifdef __CUDACC__
// AssessRegistration (odometry.cpp:604-684, the branch without robust_registration) and UpdateMap's insertion policy
// (:903-925) on v.state / v.counts; fills the rest of the verdict. One thread.
__device__ __forceinline__ void frame_policy_decide(FrameVerdict &v, const FramePolicyIn &in) {
    const IcpState &S = v.state;
    const Q4 qb{S.qb[0], S.qb[1], S.qb[2], S.qb[3]}, qe{S.qe[0], S.qe[1], S.qe[2], S.qe[3]};
    const V3 tb{S.tb[0], S.tb[1], S.tb[2]}, te{S.te[0], S.te[1], S.te[2]};
    const double ego = angular_distance_deg(qb, qe);   // EgoAngularDistance(summary.frame)
    const double rel_dist = norm(te - tb);             // summary.relative_distance (odometry.cpp:433)
    bool ok;
    if (rel_dist > in.distance_error_threshold) ok = false;
    else if (in.relative_orientation > in.orientation_error_threshold || ego > in.orientation_error_threshold) ok = false;
    else ok = !S.failed;
    bool add = true;   // UpdateMap, the branch without robust_registration
    if (in.has_insertions) add = (ego > in.insertion_ego_rotation_threshold) ? (in.skipped_enough != 0) : true;
    v.add_points_policy = add ? 1 : 0;
    if (in.do_no_insert) add = false;
    if (in.always_insert) add = true;
    int action;
    if (S.failed == 2 || S.failed == 3) action = kFrameSkip;          // the host raises an exception
    else if (!ok && in.quit_on_error) action = kFrameSkip;            // early return (odometry.cpp:437-441)
    else if (add && v.counts[1] > in.room_for) action = kFrameDeferred;
    else action = add ? kFrameInsert : kFrameEvict;
    v.assess_ok = ok ? 1 : 0;
    v.action = action;
    v.next_robust_level = 0;
    v.ego_orientation = ego;
    v.relative_distance = rel_dist;
    v.sc = slerp_consts(qb, qe);
    v.seq = in.seq;
    v.pad1 = 0;
}
// The same verdict for one attempt of the robust ladder (robust_attempt_decide). One thread.
__device__ __forceinline__ void frame_policy_decide_robust(FrameVerdict &v, const FramePolicyIn &in, const RobustPolicyIn &r) {
    const IcpState &S = v.state;
    const Q4 qb{S.qb[0], S.qb[1], S.qb[2], S.qb[3]}, qe{S.qe[0], S.qe[1], S.qe[2], S.qe[3]};
    const V3 tb{S.tb[0], S.tb[1], S.tb[2]}, te{S.te[0], S.te[1], S.te[2]};
    const RobustDecision d = robust_attempt_decide(qb, tb, qe, te, S.failed, v.counts[1], in, r);
    v.assess_ok = d.assess_ok;
    v.add_points_policy = d.add_points_policy;
    v.action = d.action;
    v.next_robust_level = d.next_robust_level;
    v.ego_orientation = d.ego_orientation;
    v.relative_distance = d.relative_distance;
    v.sc = slerp_consts(qb, qe);
    v.seq = in.seq;
    v.pad1 = 0;
}
// One warp: the verdict `v` (shared memory, complete and visible to the warp) → device memory and mapped pinned host memory,
// the sequence number last, after a system-wide fence.
__device__ __forceinline__ void frame_verdict_publish(const FrameVerdict &v, FrameVerdict *dv, FrameVerdict *hv, int lane) {
    constexpr int kWords = (int) (sizeof(FrameVerdict) / sizeof(int));
    constexpr int kSeqWord = (int) (offsetof(FrameVerdict, seq) / sizeof(int));
    const int *src = reinterpret_cast<const int *>(&v);
    int *d = reinterpret_cast<int *>(dv);
    volatile int *h = reinterpret_cast<volatile int *>(hv);
    for (int i = lane; i < kWords; i += 32) {
        d[i] = src[i];
        if (i != kSeqWord) h[i] = src[i];
    }
    __threadfence_system();
    __syncwarp();
    if (lane == 0) h[kSeqWord] = src[kSeqWord];
}
#endif

}  // namespace cticp
