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
// slam::Voxel::Coordinates (src/SlamCore/types.cxx:13-20): C int() truncation toward zero
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
#endif

}  // namespace cticp
