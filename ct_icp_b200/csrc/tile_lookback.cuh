// tile_lookback.cuh — decoupled look-back over tiles of a single pass, shared by the grid selections of the sampler
// (frame_pipeline.cu) and the map snapshot's pack / unpack (snapshot.cu).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace cticp {

// The tile publishes its own count (status 1), walks back over the tiles before it adding their counts until it meets an
// inclusive prefix (status 2), and publishes its own inclusive prefix. desc[t] = status << 32 | value, one 64-bit word, so a
// reader never sees a status without its value. A tile only waits on tiles with smaller indices, which the caller must
// guarantee are processed by CTAs that are already running (a cooperative launch taking tiles in ascending order, or tiles
// handed out in launch order from an atomic ticket).
// The walk is one warp reading a window of 32 predecessors per L2 round trip (lane j: tile end - 32 + j). The tiles of a
// launch start together, and a walk of one descriptor per trip took ~sqrt(2t) dependent trips for tile t (16 for the last
// of the 128 tiles of a 130k-point scan); a window takes at most ceil(t / 32) (3 there). The counts are integers, so every
// prefix is the one the one-descriptor walk finds. All 32 lanes of one warp; every lane returns the prefix.
__device__ __forceinline__ uint32_t tile_lookback(unsigned long long *desc, int tile, uint32_t count) {
    const int lane = threadIdx.x & 31;
    if (tile == 0) {
        if (lane == 0) atomicExch(&desc[0], (2ull << 32) | count);
        return 0u;
    }
    if (lane == 0) atomicExch(&desc[tile], (1ull << 32) | count);
    uint32_t before = 0;
    for (int end = tile;; end -= 32) {
        const int t = end - 32 + lane;
        unsigned long long d = 2ull << 32;   // before tile 0: an inclusive prefix of 0 (never the highest: tile 0 is status 2)
        if (t >= 0) {
            do d = *reinterpret_cast<volatile unsigned long long *>(&desc[t]);
            while ((uint32_t) (d >> 32) == 0u);
        }
        const uint32_t value = (uint32_t) d;
        const unsigned inclusive = __ballot_sync(0xffffffffu, (uint32_t) (d >> 32) == 2u);
        if (inclusive) {   // the highest inclusive prefix in the window plus the counts of the tiles after it
            const int hi = 31 - __clz(inclusive);
            before += __reduce_add_sync(0xffffffffu, lane >= hi ? value : 0u);
            break;
        }
        before += __reduce_add_sync(0xffffffffu, value);
    }
    if (lane == 0) atomicExch(&desc[tile], (2ull << 32) | (before + count));
    return before;
}

}  // namespace cticp
