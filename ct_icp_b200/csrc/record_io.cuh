// record_io.cuh — device reads and writes of the fields of caller-owned point records (cticp_device_scan,
// cticp_cloud_sink): x, y, z of one scalar type, one timestamp scalar of any CTICP_DTYPE_*, at any byte address.
// Shared by the kernels that pack a scan in device memory (frame_pipeline.cu) and by the trajectory transform
// (trajectory.cu).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/cticp.h"
#include "scan_pack.cuh"

namespace cticp {

// x, y, z of one record: byte-assembled (any address), natural scalar loads, or one 16-byte load (float32, 16-aligned)
enum { kLoadBytes = 0, kLoadNatural = 1, kLoadVec4 = 2 };
template <typename XT, int LOAD>
__device__ __forceinline__ void load_xyz(const unsigned char *p, XT &x, XT &y, XT &z) {
    if constexpr (LOAD == kLoadVec4) {
        const float4 v = __ldg(reinterpret_cast<const float4 *>(p));
        x = v.x; y = v.y; z = v.z;
    } else if constexpr (LOAD == kLoadNatural) {
        const XT *q = reinterpret_cast<const XT *>(p);
        x = __ldg(q); y = __ldg(q + 1); z = __ldg(q + 2);
    } else {
        x = scan_pack::load_unaligned<XT>(p);
        y = scan_pack::load_unaligned<XT>(p + sizeof(XT));
        z = scan_pack::load_unaligned<XT>(p + 2 * sizeof(XT));
    }
}
__device__ __forceinline__ double load_timestamp(const unsigned char *p, int dtype, bool aligned) {
    if (!aligned) return scan_pack::decode_timestamp(p, dtype);
    switch (dtype) {
        case CTICP_DTYPE_INT8: return (double) *reinterpret_cast<const int8_t *>(p);
        case CTICP_DTYPE_UINT8: return (double) *p;
        case CTICP_DTYPE_INT16: return (double) __ldg(reinterpret_cast<const short *>(p));
        case CTICP_DTYPE_UINT16: return (double) __ldg(reinterpret_cast<const unsigned short *>(p));
        case CTICP_DTYPE_INT32: return (double) __ldg(reinterpret_cast<const int *>(p));
        case CTICP_DTYPE_UINT32: return (double) __ldg(reinterpret_cast<const unsigned *>(p));
        case CTICP_DTYPE_FLOAT32: return (double) __ldg(reinterpret_cast<const float *>(p));
        default: return __ldg(reinterpret_cast<const double *>(p));
    }
}
// one field of a sink record: a natural store when the field is aligned to its scalar, else byte by byte
template <typename T> __device__ __forceinline__ void store_field(unsigned char *p, T v, bool aligned) {
    if (aligned) *reinterpret_cast<T *>(p) = v;
    else scan_pack::store_unaligned<T>(p, v);
}

}  // namespace cticp
