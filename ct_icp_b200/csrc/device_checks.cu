// device_checks.cu — see device_checks.h
#include "device_checks.h"

#include <cudaTypedefs.h>   // PFN_cuMemGetAddressRange (types only: the driver is reached through cudart)

#include <stdexcept>
#include <string>

#include "cuda_owner.h"

namespace cticp {

// The library links cudart statically: the driver's cuMemGetAddressRange comes through the runtime's entry-point query.
void RequireDeviceRange(const void *p, uint64_t bytes, int device, const char *what) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        throw std::invalid_argument(std::string(what) + ": not a CUDA pointer");
    }
    if ((a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) || a.device != device)
        throw std::invalid_argument(std::string(what) + ": not device memory of the handle's device");
    static PFN_cuMemGetAddressRange get_range = [] {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &fn, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            fn = nullptr;
        return reinterpret_cast<PFN_cuMemGetAddressRange>(fn);
    }();
    if (!get_range) throw CudaError("cuMemGetAddressRange is not available");
    CUdeviceptr base = 0;
    size_t size = 0;
    if (get_range(&base, &size, (CUdeviceptr) reinterpret_cast<uintptr_t>(p)) != CUDA_SUCCESS)
        throw std::invalid_argument(std::string(what) + ": not inside a device allocation");
    const uint64_t off = (uint64_t) reinterpret_cast<uintptr_t>(p) - (uint64_t) base;
    if (bytes > size || off > size - bytes)
        throw std::invalid_argument(std::string(what) + ": the described buffer extends past the end of its allocation");
}

uint64_t SpanBytes(uint64_t n, uint64_t stride, uint64_t width, const char *what) {
    uint64_t span = 0;
    if (__builtin_mul_overflow(n - 1, stride, &span) || __builtin_add_overflow(span, width, &span))
        throw std::invalid_argument(std::string(what) + ": the described buffer overflows the address space");
    return span;
}

void CheckSink(const cticp_cloud_sink &sink) {
    const size_t xs = sink.xyz_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8;
    if (sink.xyz_dtype != CTICP_DTYPE_FLOAT32 && sink.xyz_dtype != CTICP_DTYPE_FLOAT64)
        throw std::invalid_argument("sink: x/y/z must be FLOAT32 or FLOAT64");
    if (sink.t_dtype != 0 && sink.t_dtype != CTICP_DTYPE_FLOAT32 && sink.t_dtype != CTICP_DTYPE_FLOAT64)
        throw std::invalid_argument("sink: timestamp must be FLOAT32 or FLOAT64");
    if ((size_t) sink.xyz_offset + 3 * xs > sink.point_step ||
        (sink.t_dtype && (size_t) sink.t_offset + (sink.t_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8) > sink.point_step))
        throw std::invalid_argument("sink: a field lies outside the record (point_step)");
}

uint64_t SinkRecordWidth(const cticp_cloud_sink &sink) {
    const uint64_t x_end = (uint64_t) sink.xyz_offset + 3 * (sink.xyz_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8);
    const uint64_t t_end = sink.t_dtype ? (uint64_t) sink.t_offset + (sink.t_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8) : 0;
    return x_end > t_end ? x_end : t_end;
}

}  // namespace cticp
