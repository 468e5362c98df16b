// peer_exchange.cuh — the multi-GPU exchange of SURVEY §8e done by the ICP kernels themselves over NVLink peer memory.
//
// The path has exactly one exchange per Gauss-Newton iteration / LM evaluation: the sum over ranks of a 96-double
// accumulator (JTJ upper triangle, JTr, counters: 768 bytes). That is latency, not bandwidth: a library collective
// costs a kernel launch (and, inside the persistent GN kernel, would force the loop back to one launch per iteration).
// Instead every rank owns a MAILBOX in its HBM that all peers map (CUDA IPC between processes, peer access inside one
// process), and the exchanging CTA
//   1. stores its accumulator into its slot of EVERY rank's mailbox — 192 eight-byte words, each carrying 32 payload
//      bits and the 32-bit sequence number of this exchange (the "LL" idea: an aligned 8-byte store is delivered
//      atomically over NVLink, so a word whose flag matches is complete and no fence / separate flag is needed),
//   2. polls its OWN mailbox until the words of all ranks carry this exchange's sequence number,
//   3. sums the contributions in RANK ORDER — every rank adds the same numbers in the same order, so the result is
//      bit-identical everywhere and all ranks keep taking the same solver decisions (no broadcast).
// Slots are double-buffered by the parity of the sequence number: a rank can only be one exchange ahead of a peer
// (exchange n+1 needs that peer's contribution to n+1, sent after it finished reading n), so parity n is free again
// when exchange n+2 writes it. The sequence counter lives in device memory, advances by one per exchange and is the
// same number on every rank because all ranks run the same number of exchanges (same decisions, see 3.).
// A poll that does not complete within PeerLinks::timeout_cycles gives up (returns false) so a dead peer can never hang the GPU.
#pragma once
#include <cuda_runtime.h>

#include "icp.h"
#include "tagged_words.cuh"

namespace cticp {

constexpr int kMaxPeers = 8;                         // one NVSwitch domain
constexpr int kPeerWords = 2 * kAcc;                 // 8-byte words per contribution (32 payload bits each)
constexpr size_t kMailboxWords = (size_t) 2 * kMaxPeers * kPeerWords;   // [parity][source rank][word]
// Bound on the skew between ranks at an exchange, in SM cycles (PeerLinks::timeout_cycles, set by the host from
// CTICP_PEER_TIMEOUT_MS x the SM clock; default 30 s). The ranks are launched independently by their hosts: anything that
// delays one of them (a late scan, a page fault, the OS) delays the exchange, and the waiting rank must not give up on a
// healthy peer — the bound only has to be finite so that a DEAD peer cannot hang the GPU.
constexpr long long kPeerTimeoutCyclesDefault = 60000000000LL;

struct PeerLinks {
    int world = 1, rank = 0;
    unsigned long long *inbox[kMaxPeers] = {};   // inbox[p] = rank p's mailbox as mapped into THIS process (inbox[rank]: own)
    unsigned int *seq = nullptr;                 // device counter: exchanges completed so far
    long long timeout_cycles = kPeerTimeoutCyclesDefault;
};

static_assert(kMaxPeerRanks == kMaxPeers, "host / device peer tables");
inline PeerLinks PeerLinksOf(const PeerLinksHost &h) {   // the host-side description (icp.h) as a kernel argument
    PeerLinks L;
    L.world = h.world;
    L.rank = h.rank;
    for (int i = 0; i < kMaxPeers; ++i) L.inbox[i] = h.inbox[i];
    L.seq = h.seq;
    if (h.timeout_cycles > 0) L.timeout_cycles = h.timeout_cycles;
    return L;
}

// In-place sum over ranks of acc[0..kAcc) (shared memory of the calling CTA). Called by ALL threads of a CTA (any
// size that is a multiple of 32); s_half: world * kPeerWords unsigned ints of shared scratch; s_ok: one shared int.
// `seq` = sequence number of this exchange (uniform, never 0). Returns false on time-out (uniform).
__device__ __forceinline__ bool peer_allreduce(const PeerLinks &L, unsigned int seq, double *acc, unsigned int *s_half,
                                               int *s_ok) {
    const int tid = threadIdx.x, nthreads = blockDim.x;
    const size_t slot = (size_t) (seq & 1u) * kMaxPeers * kPeerWords;
    if (tid == 0) *s_ok = 1;
    __syncthreads();   // acc complete, s_ok initialised
    for (int wd = tid; wd < kPeerWords; wd += nthreads) {
        const unsigned int half = reinterpret_cast<const unsigned int *>(acc)[wd];
        const unsigned long long word = ((unsigned long long) seq << 32) | (unsigned long long) half;
        for (int p = 0; p < L.world; ++p)
            tagged_store_u64(L.inbox[p] + slot + (size_t) L.rank * kPeerWords + wd, word);
    }
    const unsigned long long *mine = L.inbox[L.rank] + slot;
    const long long t0 = clock64();
    for (int wd = tid; wd < kPeerWords; wd += nthreads) {
        for (int r = 0; r < L.world; ++r) {
            unsigned long long w = tagged_load_u64(mine + (size_t) r * kPeerWords + wd);
            while ((unsigned int) (w >> 32) != seq) {
                if (clock64() - t0 > L.timeout_cycles) {
                    *s_ok = 0;
                    break;
                }
                w = tagged_load_u64(mine + (size_t) r * kPeerWords + wd);
            }
            s_half[r * kPeerWords + wd] = (unsigned int) w;
        }
    }
    __syncthreads();
    const bool ok = *s_ok != 0;
    if (ok) {
        for (int e = tid; e < kAcc; e += nthreads) {
            double s = 0;
            for (int r = 0; r < L.world; ++r) {   // rank order: the same sum on every rank
                const unsigned int lo = s_half[r * kPeerWords + 2 * e], hi = s_half[r * kPeerWords + 2 * e + 1];
                s += __hiloint2double((int) hi, (int) lo);
            }
            acc[e] = s;
        }
    }
    __syncthreads();
    return ok;
}

}  // namespace cticp
