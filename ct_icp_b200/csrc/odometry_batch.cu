// odometry_batch.cu — one frame on each of many odometry handles in one call, the Gauss-Newton loops of the eligible
// frames in one grouped launch of k_gn_persistent (cticp_odometry_register_batch). Host code only.
#include <string>
#include <vector>

#include "engine.h"

namespace cticp {

void RegisterBatch(std::vector<BatchItem> &items) {
    std::vector<Engine::PendingFrame> frames(items.size());
    std::vector<size_t> joining;
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
            if (f.icp_pending && f.joins) joining.push_back(i);
        } catch (...) {
            it.error = std::current_exception();
        }
    }
    // one joining frame alone keeps its solo launch (the one-group case never reads a group table)
    if (joining.size() >= 2) {
        try {
            Engine &lead = *items[joining[0]].engine;
            const cudaStream_t stream = lead.Stream();
            CT_CUDA_CHECK(cudaSetDevice(lead.Device()));
            std::vector<GnProblem> problems;
            for (size_t j : joining) {
                Engine &e = *items[j].engine;
                // the launch reads every handle's keypoints, map and state: behind each one's sampling and state upload
                if (&e != &lead) CT_CUDA_CHECK(cudaStreamWaitEvent(stream, e.IcpReadyEvent(), 0));
                problems.push_back(e.IcpProblem(frames[j]));
            }
            lead.Solver().EnqueueGaussNewtonGroups(problems.data(), (int) problems.size());
            CT_CUDA_CHECK(cudaEventRecord(lead.GroupDoneEvent(), stream));
            for (size_t j : joining) items[j].engine->AdoptGroupedIcp(frames[j], lead.GroupDoneEvent(), (int) problems.size());
        } catch (...) {
            for (size_t j : joining) items[j].error = std::current_exception();
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
