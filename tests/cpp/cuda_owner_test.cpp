// csrc/cuda_owner.h on its own: what reserve leaves behind when an allocation fails, and (with a device) growth, reuse and
// moves. Prints "CUDA OWNER OK (no device)" or "CUDA OWNER OK (device)".
#include <cstdio>
#include <cstring>
#include <utility>

#include "cuda_owner.h"

using namespace cticp;

#define EXPECT(c)                                                           \
    do {                                                                    \
        if (!(c)) {                                                         \
            fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); \
            return 1;                                                       \
        }                                                                   \
    } while (0)

// f() throws a CudaError whose message names `call`
template <typename F>
static bool ThrowsNaming(F &&f, const char *call) {
    try {
        f();
    } catch (const CudaError &e) {
        return strstr(e.what(), call) != nullptr;
    }
    return false;
}

static int WithoutDevice() {
    DeviceArray<float> d;
    PinnedArray<double> h(cudaHostAllocMapped);
    for (int attempt = 0; attempt < 2; ++attempt) {   // the second reserve of the same size tries again
        EXPECT(ThrowsNaming([&] { d.reserve(1024, nullptr); }, "cudaMalloc"));
        EXPECT(d.data() == nullptr && d.capacity() == 0);
        EXPECT(ThrowsNaming([&] { h.reserve(16, nullptr); }, "cudaHostAlloc"));
        EXPECT(h.data() == nullptr && h.capacity() == 0);
    }
    Stream s;
    EXPECT(ThrowsNaming([&] { s = Stream(cudaStreamNonBlocking); }, "cudaStreamCreateWithFlags"));
    EXPECT(s.get() == nullptr);
    Event e;
    EXPECT(ThrowsNaming([&] { e = Event(cudaEventDisableTiming); }, "cudaEventCreateWithFlags"));
    EXPECT(e.get() == nullptr);
    puts("CUDA OWNER OK (no device)");
    return 0;
}

static int WithDevice() {
    Stream s(cudaStreamNonBlocking);
    EXPECT(s.get() != nullptr);
    DeviceArray<int> d;
    d.reserve(100, s.get());
    int *const first = d.data();
    EXPECT(first != nullptr && d.capacity() == 100);
    CT_CUDA_CHECK(cudaMemsetAsync(d.data(), 0, sizeof(int) * 100, s.get()));
    d.reserve(50, s.get());
    d.reserve(100, s.get());
    EXPECT(d.data() == first && d.capacity() == 100);
    d.reserve(1000, s.get());
    EXPECT(d.data() != nullptr && d.capacity() == 1000);

    DeviceArray<int> moved(std::move(d));
    EXPECT(moved.capacity() == 1000 && d.data() == nullptr && d.capacity() == 0);
    DeviceArray<int> assigned;
    assigned.reserve(4, s.get());
    assigned = std::move(moved);
    EXPECT(assigned.capacity() == 1000 && moved.data() == nullptr && moved.capacity() == 0);

    PinnedArray<double> h(cudaHostAllocMapped);
    h.reserve(8, s.get());
    h.data()[7] = 1.5;
    void *mapped = nullptr;
    CT_CUDA_CHECK(cudaHostGetDevicePointer(&mapped, h.data(), 0));
    EXPECT(mapped != nullptr);
    PinnedArray<double> h2(std::move(h));
    EXPECT(h.data() == nullptr && h.capacity() == 0 && h2.capacity() == 8 && h2.data()[7] == 1.5);

    Event e(cudaEventDisableTiming);
    CT_CUDA_CHECK(cudaEventRecord(e.get(), s.get()));
    Event e2;
    e2 = std::move(e);
    EXPECT(e2.get() != nullptr && e.get() == nullptr);
    Stream s2(std::move(s));
    EXPECT(s2.get() != nullptr && s.get() == nullptr);
    CT_CUDA_CHECK(cudaStreamSynchronize(s2.get()));
    puts("CUDA OWNER OK (device)");
    return 0;
}

int main() {
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) return WithoutDevice();
    return WithDevice();
}
