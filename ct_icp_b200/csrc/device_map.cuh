// device_map.cuh — device-resident multi-resolution voxel hash map.
//
// Replaces ct_icp::MultipleResolutionVoxelMap (include/ct_icp/map.h:99-606): tsl::robin_map<Voxel, vector<PointType>>
// becomes, per resolution, one open-addressed table of 16-byte slots {key, count} with linear probing, and one
// fixed-stride float4 point array in which slot s owns points [s*B, s*B + count).  Points are stored as fp32 offsets
// from their voxel's origin (voxel * resolution), so storage error is <= 6e-8 m at any world coordinate while all
// geometry is evaluated in fp64 (SURVEY §7 "Precision").  HBM is plentiful (80 GB): the fixed stride removes the
// allocator, the second dependent pointer load of the reference (bucket → vector → heap block) and makes a voxel's
// points one contiguous <= B*16-byte run.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "se3.cuh"

namespace cticp {

constexpr unsigned long long kEmptyKey = ~0ull;
constexpr unsigned long long kTombKey = ~0ull - 1ull;
constexpr int kVoxelBias = 1 << 20;   // |voxel coordinate| < 2^20
constexpr int kNil = -1;

struct __align__(16) MapSlot {
    unsigned long long key;
    uint32_t count;
    uint32_t _pad;
};

struct MapLevel {
    MapSlot *slots;       // [cap]
    float4 *points;       // [cap * B]  xyz = offset from voxel origin, w = +-(source frame ordinal + 1): the sign says
                          //            whether this point's copy of the voxel normal is flipped (map.h:222-226)
    int *head;            // [cap] insertion scratch: per-voxel candidate list head (kNil between inserts)
    double *normals;      // [cap * 4] or nullptr: voxel normal (x, y, z) and 1.0 once computed (PointType::normal /
                          //            is_normal_computed, map.h:211-235); only kept when a search may filter on it
    uint32_t cap_mask;    // cap - 1 (cap is a power of two)
    int B;                // max_num_points
    double res;           // resolution
    double min_dist2;     // min_distance_between_points^2
};

struct MapCounters {   // device-resident, one per level
    unsigned long long num_points;
    unsigned int num_voxels;
    unsigned int num_tombs;
    unsigned int num_touched;
    unsigned int overflow;   // set when a probe sequence wrapped (table full)
};

CT_HD unsigned long long pack_voxel(int x, int y, int z) {
    return ((unsigned long long) (unsigned) (x + kVoxelBias) << 42) | ((unsigned long long) (unsigned) (y + kVoxelBias) << 21) |
           (unsigned long long) (unsigned) (z + kVoxelBias);
}
CT_HD void unpack_voxel(unsigned long long k, int &x, int &y, int &z) {
    x = int((k >> 42) & 0x1FFFFF) - kVoxelBias;
    y = int((k >> 21) & 0x1FFFFF) - kVoxelBias;
    z = int(k & 0x1FFFFF) - kVoxelBias;
}
CT_HD uint32_t hash_key(unsigned long long k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return (uint32_t) k;
}
// slam::Voxel::Coordinates (src/SlamCore/types.cxx:13-20): C int() truncation toward zero (on the device a quotient beyond
// the int range saturates, so such a query fails stencil_in_range)
CT_HD int voxel_coord(double p, double res) { return int(p / res); }
// the same integer from p * (1 / res): the product is within 2 ulp of the quotient, so the truncation can only differ when
// the quotient is within ~1e-15 relative of an integer — those (and only those) take the division. Three fp64 divisions
// (~30 dependent instructions each) leave the serial lane-per-keypoint phase of the gathers.
CT_HD int voxel_coord_rcp(double p, double res, double inv_res) {
    const double q = p * inv_res;
#ifdef __CUDA_ARCH__
    const int k = f64_trunc(q);                       // (conversions off the XU pipe, se3.cuh)
    const double f = fabs(q - i32_to_f64(k));
#else
    const int k = int(q);
    const double f = fabs(q - (double) k);
#endif
    const double guard = 1e-12 * (1.0 + fabs(q));
    return (f < guard || f > 1.0 - guard) ? int(p / res) : k;
}

// A key holds 21 bits per axis: voxel coordinates in [-2^20, 2^20). slam::Voxel is an int, so the map skips what it cannot
// key instead of letting a coordinate wrap onto a voxel on the far side of the range (or onto kEmptyKey).
constexpr double kVoxelCoordLimit = 2097152.0;   // 2^21: a quotient |p / res| beyond it is out of range (and voxel_coord_rcp
                                                 // converts only |p / res| < 2^31)
CT_HD bool voxel_in_range(int v) { return v >= -kVoxelBias && v < kVoxelBias; }
// the key of a point's voxel; false: a non-finite coordinate, or a voxel coordinate outside [-2^20, 2^20)
CT_HD bool voxel_key(double x, double y, double z, double res, double inv_res, unsigned long long &key) {
    if (!(fabs(x * inv_res) < kVoxelCoordLimit) || !(fabs(y * inv_res) < kVoxelCoordLimit) ||
        !(fabs(z * inv_res) < kVoxelCoordLimit))
        return false;
    const int vx = voxel_coord_rcp(x, res, inv_res), vy = voxel_coord_rcp(y, res, inv_res), vz = voxel_coord_rcp(z, res, inv_res);
    if (!voxel_in_range(vx) || !voxel_in_range(vy) || !voxel_in_range(vz)) return false;
    key = pack_voxel(vx, vy, vz);
    return true;
}
// a query's voxel coordinate: voxel_coord_rcp, or +-2^21 (outside the range) when |p / res| >= 2^21
CT_HD int query_voxel_coord(double p, double res, double inv_res) {
    const double q = p * inv_res;
    if (fabs(q) >= kVoxelCoordLimit) return q < 0.0 ? -2 * kVoxelBias : 2 * kVoxelBias;
    return voxel_coord_rcp(p, res, inv_res);
}
// whether the (2r+1)^3 stencil around voxel (kx, ky, kz) lies inside [-2^20, 2^20) on every axis. Checked once per query:
// a query whose stencil leaves the range finds no neighbours, since its out-of-range keys would alias stored voxels.
CT_HD bool stencil_in_range(int kx, int ky, int kz, int r) {
    const int lo = -kVoxelBias + r, hi = kVoxelBias - 1 - r;
    return kx >= lo && kx <= hi && ky >= lo && ky <= hi && kz >= lo && kz <= hi;
}
// the x coordinate a query whose stencil leaves the range is given (r < 2^20): every stencil key then has x + 2^20 in
// [2^21, 2^22), so bit 63 set, which no stored key has; such a query finds nothing with the gather left as it is
constexpr int kVoxelNowhere = 2 * kVoxelBias;
CT_HD void confine_query(int &kx, int ky, int kz, int r) {
    if (!stencil_in_range(kx, ky, kz, r)) kx = kVoxelNowhere;
}

#ifdef __CUDACC__
// Lookup: returns slot index or -1. Linear probing, stops at the first empty slot; tombstones are skipped.
__device__ __forceinline__ int map_find(const MapLevel &L, unsigned long long key, uint32_t *count_out) {
    uint32_t h = hash_key(key) & L.cap_mask;
    for (uint32_t probe = 0; probe <= L.cap_mask; ++probe) {
        // one 16-byte load: key + count
        const uint4 raw = __ldg(reinterpret_cast<const uint4 *>(L.slots + h));
        unsigned long long k = (unsigned long long) raw.x | ((unsigned long long) raw.y << 32);
        if (k == key) {
            *count_out = raw.z;
            return (int) h;
        }
        if (k == kEmptyKey) return -1;
        h = (h + 1) & L.cap_mask;
    }
    return -1;
}

// -DCTICP_DEBUG_TIMERS builds: phase stamps of the fused sampler and the fused map update. Slot 0 takes the earliest start of
// a CTA, every other slot the latest end of one phase over the CTAs, all in %globaltimer ns (comparable across SMs, unlike
// clock64; a few reads per CTA and launch cost nothing, unlike the per-iteration reads icp.h warns about). The host prints
// them per launch when the environment has CTICP_DEBUG_TIMERS. Default builds compile none of this.
#ifdef CTICP_DEBUG_TIMERS
constexpr int kPhaseSlots = 16;
__device__ __forceinline__ unsigned long long phase_clock() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void phase_begin(unsigned long long *stamps) {
    if (threadIdx.x == 0) atomicMin(stamps, phase_clock());
}
// every thread of the CTA
__device__ __forceinline__ void phase_end(unsigned long long *stamps, int slot) {
    __syncthreads();
    if (threadIdx.x == 0) atomicMax(stamps + slot, phase_clock());
}
#define PHASE_STAMP(...) __VA_ARGS__
#else
#define PHASE_STAMP(...)
#endif
#endif

}  // namespace cticp
