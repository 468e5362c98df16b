// cuda_owner.h — move-only owners of CUDA allocations, streams and events, and the one CT_CUDA_CHECK.
// Host-only: compiles with a plain C++ compiler against cuda_runtime.h. Destructors never throw and ignore release errors.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <stdexcept>
#include <string>
#include <utility>

namespace cticp {

struct CudaError : std::runtime_error {
    using std::runtime_error::runtime_error;
};

#define CT_CUDA_CHECK(expr)                                                                              \
    do {                                                                                                 \
        cudaError_t _e = (expr);                                                                         \
        if (_e != cudaSuccess)                                                                           \
            throw ::cticp::CudaError(std::string(#expr) + ": " + cudaGetErrorString(_e) + " @" + __FILE__ + \
                                     ":" + std::to_string(__LINE__));                                    \
    } while (0)

// One grow-only allocation of T: cudaMalloc, or cudaHostAlloc with the flags given at construction when kPinned.
// reserve(n, stream) does nothing while n <= capacity(); otherwise it synchronises `stream` before freeing what it
// holds, and records the new pointer and capacity only once the allocation succeeded: after a failure the holder is
// empty, so the next reserve allocates again instead of reusing a freed pointer.
template <typename T, bool kPinned>
class CudaArray {
public:
    CudaArray() = default;
    explicit CudaArray(unsigned int host_alloc_flags) : flags_(host_alloc_flags) {}
    ~CudaArray() { clear(); }
    CudaArray(CudaArray &&o) noexcept
        : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)), flags_(o.flags_) {}
    CudaArray &operator=(CudaArray &&o) noexcept {
        if (this != &o) {
            clear();
            p_ = std::exchange(o.p_, nullptr);
            n_ = std::exchange(o.n_, 0);
            flags_ = o.flags_;
        }
        return *this;
    }
    CudaArray(const CudaArray &) = delete;
    CudaArray &operator=(const CudaArray &) = delete;

    T *data() const { return p_; }
    size_t capacity() const { return n_; }

    void reserve(size_t n, cudaStream_t stream) {
        if (n <= n_) return;
        if (p_) {
            CT_CUDA_CHECK(cudaStreamSynchronize(stream));
            clear();
        }
        void *p = nullptr;
        if constexpr (kPinned)
            CT_CUDA_CHECK(cudaHostAlloc(&p, sizeof(T) * n, flags_));
        else
            CT_CUDA_CHECK(cudaMalloc(&p, sizeof(T) * n));
        p_ = static_cast<T *>(p);
        n_ = n;
    }
    // frees now, without synchronising: the caller orders this after the work that uses the memory
    void clear() {
        if (p_) {
            if constexpr (kPinned)
                cudaFreeHost(p_);
            else
                cudaFree(p_);
        }
        p_ = nullptr;
        n_ = 0;
    }

private:
    T *p_ = nullptr;
    size_t n_ = 0;
    unsigned int flags_ = cudaHostAllocDefault;
};

template <typename T>
using DeviceArray = CudaArray<T, false>;
template <typename T>
using PinnedArray = CudaArray<T, true>;

// One cudaStream_t / cudaEvent_t: empty when default-constructed, created with `flags` otherwise.
template <typename H, cudaError_t (*Destroy)(H)>
class CudaHandle {
public:
    CudaHandle() = default;
    ~CudaHandle() {
        if (h_) Destroy(h_);
    }
    CudaHandle(CudaHandle &&o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
    CudaHandle &operator=(CudaHandle &&o) noexcept {
        if (this != &o) {
            if (h_) Destroy(h_);
            h_ = std::exchange(o.h_, nullptr);
        }
        return *this;
    }
    CudaHandle(const CudaHandle &) = delete;
    CudaHandle &operator=(const CudaHandle &) = delete;

    H get() const { return h_; }

protected:
    H h_ = nullptr;
};

class Stream : public CudaHandle<cudaStream_t, cudaStreamDestroy> {
public:
    Stream() = default;
    explicit Stream(unsigned int flags) {
        cudaStream_t s = nullptr;
        CT_CUDA_CHECK(cudaStreamCreateWithFlags(&s, flags));
        h_ = s;
    }
};

class Event : public CudaHandle<cudaEvent_t, cudaEventDestroy> {
public:
    Event() = default;
    explicit Event(unsigned int flags) {
        cudaEvent_t e = nullptr;
        CT_CUDA_CHECK(cudaEventCreateWithFlags(&e, flags));
        h_ = e;
    }
};

}  // namespace cticp
