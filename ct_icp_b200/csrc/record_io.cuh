// record_io.cuh — device reads and writes of the fields of caller-owned point records (cticp_device_scan,
// cticp_cloud_sink): x, y, z of one scalar type, one timestamp scalar of any CTICP_DTYPE_*, at any byte address.
// Shared by the kernels that pack a scan in device memory (frame_pipeline.cu) and by the trajectory transform
// (trajectory.cu).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/cticp.h"
#include "scan_pack.cuh"
#include "se3.cuh"

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

// a cticp_cloud_sink as the generators' kernels write it (synthetic.cu, lidar_sim.cu): x, y, z as FLOAT32 (rounded to
// nearest) or FLOAT64, the timestamp as FLOAT32, FLOAT64 or not at all
struct GenSink {
    unsigned char *data;
    uint64_t cap;
    uint32_t step, xoff, toff;
    int xdt, tdt, x_aligned, t_aligned, world;
};

__device__ __forceinline__ void store_gen_record(const GenSink &s, uint64_t pos, const V3 &p, double t) {
    unsigned char *rec = s.data + pos * s.step;
    if (s.xdt == CTICP_DTYPE_FLOAT32) {
        store_field<float>(rec + s.xoff, scan_pack::hi_of(p.x), s.x_aligned);
        store_field<float>(rec + s.xoff + 4, scan_pack::hi_of(p.y), s.x_aligned);
        store_field<float>(rec + s.xoff + 8, scan_pack::hi_of(p.z), s.x_aligned);
    } else {
        store_field<double>(rec + s.xoff, p.x, s.x_aligned);
        store_field<double>(rec + s.xoff + 8, p.y, s.x_aligned);
        store_field<double>(rec + s.xoff + 16, p.z, s.x_aligned);
    }
    if (s.tdt == CTICP_DTYPE_FLOAT32) store_field<float>(rec + s.toff, scan_pack::hi_of(t), s.t_aligned);
    else if (s.tdt == CTICP_DTYPE_FLOAT64) store_field<double>(rec + s.toff, t, s.t_aligned);
}

inline GenSink MakeGenSink(unsigned char *data, const cticp_cloud_sink &sink, uint64_t cap) {
    GenSink sa{};
    sa.data = data;
    sa.cap = cap;
    sa.step = sink.point_step;
    sa.xoff = sink.xyz_offset;
    sa.toff = sink.t_offset;
    sa.xdt = sink.xyz_dtype;
    sa.tdt = sink.t_dtype;
    sa.world = sink.world ? 1 : 0;
    if (data) {
        const size_t osz = sink.xyz_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8, otsz = sink.t_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8;
        sa.x_aligned = ((reinterpret_cast<uintptr_t>(data) + sink.xyz_offset) % osz == 0 && sink.point_step % osz == 0);
        sa.t_aligned = ((reinterpret_cast<uintptr_t>(data) + sink.t_offset) % otsz == 0 && sink.point_step % otsz == 0);
    }
    return sa;
}

}  // namespace cticp
