// odometry_batch.cu — one frame on each of many odometry handles in one call, the ICP loops of the eligible frames in one
// grouped launch per kind: solver GN in k_gn_persistent, each k_lm_persistent mode (CERES nearest neighbour, CERES
// distance-based, ROBUST) in k_lm_persistent (cticp_odometry_register_batch). The attempts of robust registrations run
// in rounds, in kinds of their own. Host code only.
#include <string>
#include <vector>

#include "engine.h"

namespace cticp {

namespace {

// One grouped launch per kind over the frames of `joining`, on the stream of each kind's first joining handle. A
// joining frame alone in its kind keeps its solo launch (the one-group case never reads a group table).
void LaunchGroups(std::vector<BatchItem> &items, std::vector<Engine::PendingFrame> &frames,
                  const std::vector<size_t> (&joining)[Engine::kJoinKinds]) {
    for (int kind = 0; kind < Engine::kJoinKinds; ++kind) {
        const std::vector<size_t> &J = joining[kind];
        if (J.size() < 2) continue;
        try {
            Engine &lead = *items[J[0]].engine;
            const cudaStream_t stream = lead.Stream();
            // the launch reads every handle's keypoints, map, state and (LM) buffers: behind each one's sampling, state
            // upload and buffer preparation
            const auto wait_for = [&](Engine &e) {
                CT_CUDA_CHECK(cudaSetDevice(lead.Device()));
                if (&e != &lead) CT_CUDA_CHECK(cudaStreamWaitEvent(stream, e.IcpReadyEvent(), 0));
            };
            if (kind == Engine::kJoinsGn || kind == Engine::kJoinsLadderGn) {
                std::vector<GnProblem> problems;
                for (size_t j : J) {
                    Engine &e = *items[j].engine;
                    wait_for(e);
                    problems.push_back(e.IcpProblem(frames[j]));
                }
                lead.Solver().EnqueueGaussNewtonGroups(problems.data(), (int) problems.size());
            } else {
                std::vector<LmProblem> problems;
                for (size_t j : J) {
                    Engine &e = *items[j].engine;
                    problems.push_back(e.CeresProblem(frames[j]));   // (on e's stream, before the wait)
                    wait_for(e);
                }
                lead.Solver().EnqueueCeresGroups(problems.data(), (int) problems.size());
            }
            CT_CUDA_CHECK(cudaEventRecord(lead.GroupDoneEvent(), stream));
            for (size_t j : J) items[j].engine->AdoptGroupedIcp(frames[j], lead.GroupDoneEvent(), (int) J.size());
        } catch (...) {
            for (size_t j : J) items[j].error = std::current_exception();
        }
    }
}

}  // namespace

void RegisterBatch(std::vector<BatchItem> &items) {
    std::vector<Engine::PendingFrame> frames(items.size());
    std::vector<size_t> joining[Engine::kJoinKinds];
    std::vector<size_t> ladder;   // robust registrations with an attempt pending
    // phase 1 on every handle: each stops before its (first attempt's) ICP launch
    for (size_t i = 0; i < items.size(); ++i) {
        BatchItem &it = items[i];
        try {
            Engine::PendingFrame &f = frames[i];
            switch (it.kind) {
                case CTICP_BATCH_HOST:
                    it.engine->BeginFrame(it.scan, it.frame_id, it.initial_estimate, it.out, it.motion_model, f);
                    break;
                case CTICP_BATCH_DEVICE:
                    it.engine->BeginDevice(it.scan, it.producer, it.frame_id, it.initial_estimate, it.out, it.motion_model, f);
                    break;
                default:
                    it.engine->BeginStaged(it.slot, it.frame_id, it.out, f);
            }
            if (f.icp_pending && f.joins != Engine::kJoinsNone) joining[f.joins].push_back(i);
            if (f.ladder && f.icp_pending) ladder.push_back(i);
        } catch (...) {
            it.error = std::current_exception();
        }
    }
    // phase 2, round 0: the grouped launches of the plain frames and of every robust registration's first attempt
    LaunchGroups(items, frames, joining);
    // phase 3 of the plain frames, item by item (a frame that does not join launches its own ICP now)
    for (size_t i = 0; i < items.size(); ++i) {
        if (items[i].error || frames[i].ladder) continue;
        try {
            items[i].engine->CompleteFrame(frames[i]);
        } catch (...) {
            items[i].error = std::current_exception();
        }
    }
    // the robust ladders in rounds: round r has launched attempt r of every frame still in `ladder`. Every handle enqueues
    // its tail, then the host takes the verdicts; a rejected frame has begun its next attempt and joins round r + 1. Each
    // ladder ends by its own last allowed attempt, so the rounds are bounded by the largest robust_num_attempts.
    while (!ladder.empty()) {
        const auto fail = [&](size_t i) { items[i].error = std::current_exception(); };
        for (size_t i : ladder) {
            if (items[i].error) continue;
            try {
                items[i].engine->LaunchPending(frames[i]);   // (solo: not in a grouped launch of this round)
            } catch (...) {
                fail(i);
            }
        }
        for (size_t i : ladder) {
            if (items[i].error) continue;
            try {
                items[i].engine->EnqueueTail();
            } catch (...) {
                fail(i);
            }
        }
        std::vector<size_t> next;
        for (auto &J : joining) J.clear();
        for (size_t i : ladder) {
            if (items[i].error) continue;
            try {
                Engine::PendingFrame &f = frames[i];
                items[i].engine->EndAttempt(f);
                if (f.ladder_accepted) {
                    items[i].engine->CompleteFrame(f);   // FinishFrame
                    continue;
                }
                next.push_back(i);
                if (f.joins != Engine::kJoinsNone) joining[f.joins].push_back(i);
            } catch (...) {
                fail(i);
            }
        }
        ladder.swap(next);
        LaunchGroups(items, frames, joining);
    }
}

}  // namespace cticp
