// tagged_words.cuh — hand-off of small payloads between CTAs without fences or flags (NCCL's "LL" idea).
// Every aligned 8-byte word carries 32 payload bits in its low half and a 32-bit tag in its high half. An aligned 8-byte
// store is seen whole or not at all, so a reader that finds the tag it expects has the payload of that store: no fence
// between payload and flag, no separate flag word, one memory round trip per hand-off. Tags must never repeat while a
// stale word could still be read with them (the users keep a counter and zero the words when it would wrap).
// Users: the NVLink peer mailboxes (peer_exchange.cuh) and the loop of k_gn_persistent (icp_gn.cu).
#pragma once
#include <cuda_runtime.h>

namespace cticp {

__device__ __forceinline__ void tagged_store_u64(unsigned long long *p, unsigned long long v) {
    asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long tagged_load_u64(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
// two words at a 16-byte aligned address in one access (each word on its own is still the unit of completeness)
__device__ __forceinline__ void tagged_store_u64x2(unsigned long long *p, unsigned long long a, unsigned long long b) {
    asm volatile("st.volatile.global.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"(a), "l"(b) : "memory");
}
__device__ __forceinline__ ulonglong2 tagged_load_u64x2(const unsigned long long *p) {
    ulonglong2 v;
    asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ unsigned long long tagged_word(unsigned int tag, unsigned int payload) {
    return ((unsigned long long) tag << 32) | (unsigned long long) payload;
}
__device__ __forceinline__ unsigned int word_tag(unsigned long long w) { return (unsigned int) (w >> 32); }
__device__ __forceinline__ unsigned int word_payload(unsigned long long w) { return (unsigned int) w; }
// both words of a pair carry `tag`
__device__ __forceinline__ bool pair_tagged(ulonglong2 v, unsigned int tag) {
    return word_tag(v.x) == tag && word_tag(v.y) == tag;
}
// a double as two tagged words (low half first, the order of its bytes in memory) and back: exact for every bit pattern
__device__ __forceinline__ void tagged_store_double(unsigned long long *p, unsigned int tag, double d) {
    tagged_store_u64x2(p, tagged_word(tag, (unsigned int) __double2loint(d)), tagged_word(tag, (unsigned int) __double2hiint(d)));
}
__device__ __forceinline__ double pair_double(ulonglong2 v) {
    return __hiloint2double((int) word_payload(v.y), (int) word_payload(v.x));
}

}  // namespace cticp
