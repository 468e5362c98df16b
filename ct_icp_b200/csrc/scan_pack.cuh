// scan_pack.cuh — the packing format of a scan, shared by the host loops (engine.cu) and the device kernels of a scan in
// GPU memory (frame_pipeline.cu):
//   alpha = spans ? (t - mn) * inv : 1        (GetAlphaTimestamp w.r.t. the pose pair, include/SlamCore/types.h:192-219)
//   hi    = float of x, y, z, alpha           (the float4 every kernel reads)
//   lo    = value - (double) (float) value    (the residual plane, load_raw in se3.cuh)
//   a float64 scan "needs lo" when some coordinate is not float32-representable
// and the timestamps written back: mn + alpha * (mx - mn).
//
// The device branches spell every operation with an explicit rounding intrinsic: nvcc contracts a * b + c into an FMA by
// default, and the device results must be the host's bit for bit. Compiles with plain g++ (tests/cpp/scan_pack_test.cpp).
#pragma once
#include <cstdint>
#include <cstring>

#ifdef __CUDACC__
#define SP_HD __host__ __device__ __forceinline__
#else
#define SP_HD inline
#endif

namespace cticp {
namespace scan_pack {

// CTICP_DTYPE_* → bytes (0: unknown)
SP_HD unsigned dtype_size(int dtype) {
    switch (dtype) {
        case 1: case 2: return 1;
        case 3: case 4: return 2;
        case 5: case 6: case 7: return 4;
        case 8: return 8;
        default: return 0;
    }
}

// A scalar at any byte address (PointCloud2 records are packed: no alignment promise). The device assembles it from bytes:
// a misaligned 4- or 8-byte load faults on the GPU.
template <typename T> SP_HD T load_unaligned(const void *p) {
    T v;
#ifdef __CUDA_ARCH__
    const unsigned char *b = static_cast<const unsigned char *>(p);
    unsigned long long u = 0;
#pragma unroll
    for (unsigned k = 0; k < sizeof(T); ++k) u |= (unsigned long long) b[k] << (8 * k);
    if constexpr (sizeof(T) == 8) {
        memcpy(&v, &u, 8);
    } else {
        const unsigned w = (unsigned) u;
        memcpy(&v, &w, sizeof(T));
    }
#else
    memcpy(&v, p, sizeof(T));
#endif
    return v;
}
template <typename T> SP_HD void store_unaligned(void *p, T v) {
#ifdef __CUDA_ARCH__
    unsigned char *b = static_cast<unsigned char *>(p);
    unsigned long long u = 0;
    memcpy(&u, &v, sizeof(T));
#pragma unroll
    for (unsigned k = 0; k < sizeof(T); ++k) b[k] = (unsigned char) (u >> (8 * k));
#else
    memcpy(p, &v, sizeof(T));
#endif
}

// static_cast<double> of the timestamp scalar at p (any CTICP_DTYPE_*; unknown dtypes are rejected before this is reached)
SP_HD double decode_timestamp(const void *p, int dtype) {
    switch (dtype) {
        case 1: return (double) load_unaligned<int8_t>(p);
        case 2: return (double) load_unaligned<uint8_t>(p);
        case 3: return (double) load_unaligned<int16_t>(p);
        case 4: return (double) load_unaligned<uint16_t>(p);
        case 5: return (double) load_unaligned<int32_t>(p);
        case 6: return (double) load_unaligned<uint32_t>(p);
        case 7: return (double) load_unaligned<float>(p);
        default: return load_unaligned<double>(p);
    }
}

// one step of the timestamp min / max: NaN compares false both ways and is skipped
SP_HD double min_step(double m, double t) { return t < m ? t : m; }
SP_HD double max_step(double m, double t) { return t > m ? t : m; }

// The pose pair's timestamps → the constants of alpha (std::min / std::max argument order kept)
struct AlphaRange {
    double mn, mx, inv;
    bool spans;
};
SP_HD AlphaRange alpha_range(double begin_ts, double end_ts) {
    AlphaRange r;
    r.mn = (end_ts < begin_ts) ? end_ts : begin_ts;
    r.mx = (begin_ts < end_ts) ? end_ts : begin_ts;
    r.spans = r.mx > r.mn;
#ifdef __CUDA_ARCH__
    r.inv = r.spans ? __ddiv_rn(1.0, __dsub_rn(r.mx, r.mn)) : 0.0;
#else
    r.inv = r.spans ? 1.0 / (r.mx - r.mn) : 0.0;
#endif
    return r;
}
SP_HD double alpha_of(double t, const AlphaRange &r) {
#ifdef __CUDA_ARCH__
    return r.spans ? __dmul_rn(__dsub_rn(t, r.mn), r.inv) : 1.0;
#else
    return r.spans ? (t - r.mn) * r.inv : 1.0;
#endif
}

SP_HD float hi_of(float v) { return v; }
SP_HD float hi_of(double v) {
#ifdef __CUDA_ARCH__
    return __double2float_rn(v);
#else
    return (float) v;
#endif
}
SP_HD float lo_of(double v) {
#ifdef __CUDA_ARCH__
    return __double2float_rn(__dsub_rn(v, (double) __double2float_rn(v)));
#else
    return (float) (v - (double) (float) v);
#endif
}
SP_HD bool needs_lo(float) { return false; }
SP_HD bool needs_lo(double v) { return (double) hi_of(v) != v; }

// a coordinate rebuilt from its planes: hi (+ lo when the scan has a residual plane)
SP_HD double rebuild(float hi, float lo, bool has_lo) {
#ifdef __CUDA_ARCH__
    return has_lo ? __dadd_rn((double) hi, (double) lo) : (double) hi;
#else
    return has_lo ? (double) hi + (double) lo : (double) hi;
#endif
}
// the timestamp of a packed point: mn + alpha * (mx - mn), alpha = hi + (lo or 0)
SP_HD double timestamp_of(float alpha_hi, float alpha_lo, bool has_lo, double mn, double mx) {
#ifdef __CUDA_ARCH__
    const double a = __dadd_rn((double) alpha_hi, has_lo ? (double) alpha_lo : 0.0);
    return __dadd_rn(mn, __dmul_rn(a, __dsub_rn(mx, mn)));
#else
    const double a = (double) alpha_hi + (has_lo ? (double) alpha_lo : 0.0);
    return mn + a * (mx - mn);
#endif
}

}  // namespace scan_pack
}  // namespace cticp
