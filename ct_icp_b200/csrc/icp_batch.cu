// icp_batch.cu — CTA policy of the persistent registration kernels (EnqueueGaussNewtonGroups, icp_gn.cu;
// EnqueueCeresGroups, icp_lm.cu). Host code only.
#include <algorithm>
#include <vector>

#include "icp.h"

namespace cticp {

int GatherBlocks(size_t k_hint, int max_blocks, int kp_per_cta) {
    // One CTA (kGatherWarps warps, 128 registers per thread) per SM. A keypoint set smaller than the machine is spread
    // thin — `kp_per_cta` keypoints per CTA, so each keypoint's warp has an SM sub-partition nearly to itself: the loop
    // is latency-bound there — until every SM has a CTA; beyond that the tiles widen (gn_gather_tiles).
    // k_hint is an ESTIMATE of the keypoint count (the exact count lives on the device): too small only widens the
    // tiles, too large only adds idle CTAs whose zero partials have to be summed.
    size_t want = (k_hint + kp_per_cta - 1) / kp_per_cta;
    return (int) std::max<size_t>(1, std::min(want, (size_t) max_blocks));
}

// CTA policy of a batched persistent launch: gather[b] = the gather (GN) / worker (LM) CTAs of problem b (each problem also
// has its solver CTA). Contract:
//  - When every problem fits with what a solo call would give it — solo_b = GatherBlocks(n_b + 16, coresident - 1), the
//    grid of EnqueueGaussNewton and of EnqueueCeres's persistent launch for n_b = k_upper / k_hint — and Σ (1 + solo_b) <= coresident,
//    gather[b] = solo_b. Keypoint ranges, tiles and the order of every reduction are then those of the solo call: each
//    problem's result is bit-identical to it.
//  - Otherwise the coresident - batch CTAs left for gathering are dealt one at a time to the problem with the most keypoints
//    per gather CTA (exact integer comparison, ties to the lower index), starting from 1 each and never beyond solo_b. The
//    busiest CTA sets a group's iteration time, so this balances the groups. The result then differs from the solo call's
//    by summation order only, and is a function of (n, coresident): bit-reproducible run to run.
// Requires 2 * batch <= coresident.
void BatchGatherCtas(const size_t *n, int batch, int coresident, int kp_per_cta, int *gather) {
    long long total = 0;
    std::vector<int> solo(batch);
    for (int b = 0; b < batch; ++b) {
        solo[b] = GatherBlocks(n[b] + 16, std::max(1, coresident - 1), kp_per_cta);
        total += 1 + solo[b];
    }
    if (total <= coresident) {
        for (int b = 0; b < batch; ++b) gather[b] = solo[b];
        return;
    }
    for (int b = 0; b < batch; ++b) gather[b] = 1;
    for (int left = coresident - 2 * batch; left > 0; --left) {
        int best = -1;
        for (int b = 0; b < batch; ++b) {
            if (gather[b] >= solo[b]) continue;
            // n_b / gather_b > n_best / gather_best
            if (best < 0 || (unsigned long long) n[b] * gather[best] > (unsigned long long) n[best] * gather[b]) best = b;
        }
        if (best < 0) break;
        gather[best] += 1;
    }
}

}  // namespace cticp
