// odometry_batch.cu — one frame on each of many odometry handles in one call, the ICP loops of the eligible frames in one
// grouped launch per kind: solver GN in k_gn_persistent, each k_lm_persistent mode (CERES nearest neighbour, CERES
// distance-based, ROBUST) in k_lm_persistent (cticp_odometry_register_batch). Host code only.
#include <string>
#include <vector>

#include "engine.h"

namespace cticp {

void RegisterBatch(std::vector<BatchItem> &items) {
    std::vector<Engine::PendingFrame> frames(items.size());
    std::vector<size_t> joining[Engine::kJoinKinds];
    // phase 1 on every handle: each stops before its ICP launch (a frame that does not join launches its own now)
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
        } catch (...) {
            it.error = std::current_exception();
        }
    }
    // phase 2: one grouped launch per kind, on the stream of its first joining handle. A joining frame alone in its kind
    // keeps its solo launch (the one-group case never reads a group table).
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
            if (kind == Engine::kJoinsGn) {
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
    // phase 3, item by item
    for (size_t i = 0; i < items.size(); ++i) {
        if (items[i].error) continue;
        try {
            items[i].engine->CompleteFrame(frames[i]);
        } catch (...) {
            items[i].error = std::current_exception();
        }
    }
}

}  // namespace cticp
