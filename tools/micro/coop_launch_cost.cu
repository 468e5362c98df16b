// Micro-benchmark: what does a cooperative launch cost on the device timeline, next to a plain launch of the same grid?
// Chains of N dependent short kernels on one stream, timed with events; grid = 4 CTAs per SM (all SMs) x 256 threads, each kernel
// with `syncs` grid-wide barriers — cg::grid.sync() under cudaLaunchCooperativeKernel vs a hand-rolled arrive/epoch
// barrier under a plain launch (all CTAs co-resident by construction).
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o coop_launch_cost coop_launch_cost.cu ; run: ./coop_launch_cost
#include <cooperative_groups.h>
#include <cstdio>
#include <cuda_runtime.h>
namespace cg = cooperative_groups;

__device__ __forceinline__ void soft_barrier(unsigned int *words) {
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int epoch = *((volatile unsigned int *) (words + 1));
        __threadfence();
        if (atomicAdd(words, 1u) == gridDim.x - 1) {
            words[0] = 0;
            __threadfence();
            atomicAdd(words + 1, 1u);
        } else {
            const long long t0 = clock64();
            while (*((volatile unsigned int *) (words + 1)) == epoch)
                if (clock64() - t0 > 400000000LL) break;   // bounded: a protocol error ends the kernel instead of hanging the GPU
        }
        __threadfence();
    }
    __syncthreads();
}

__global__ void k_coop(int syncs, float *out) {
    cg::grid_group grid = cg::this_grid();
    float v = threadIdx.x;
    for (int i = 0; i < syncs; ++i) {
        v = v * 1.0001f + 1.f;
        grid.sync();
    }
    if (v == -1.f) out[0] = v;
}
__global__ void k_soft(int syncs, float *out, unsigned int *words) {
    float v = threadIdx.x;
    for (int i = 0; i < syncs; ++i) {
        v = v * 1.0001f + 1.f;
        soft_barrier(words);
    }
    if (v == -1.f) out[0] = v;
}
__global__ void k_plain(float *out) {
    float v = threadIdx.x * 1.0001f;
    if (v == -1.f) out[0] = v;
}

int main() {
    float *out;
    unsigned int *words;
    cudaMalloc(&out, 4);
    cudaMalloc(&words, 8);
    cudaMemset(words, 0, 8);
    cudaStream_t s;
    cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    const int chain = 30;
    for (int per_sm : {1, 4}) {
        const int grid = per_sm * sms;
        for (int syncs : {0, 1, 6}) {
            for (int mode = 0; mode < 3; ++mode) {   // 0 plain launch no barrier, 1 cooperative + grid.sync, 2 plain + soft barrier
                if (mode == 0 && syncs != 0) continue;
                float best = 1e9f;
                for (int rep = 0; rep < 5; ++rep) {
                    cudaEventRecord(e0, s);
                    for (int i = 0; i < chain; ++i) {
                        if (mode == 0) k_plain<<<grid, 256, 0, s>>>(out);
                        else if (mode == 1) {
                            void *args[] = {(void *) &syncs, (void *) &out};
                            cudaLaunchCooperativeKernel((void *) k_coop, dim3(grid), dim3(256), args, 0, s);
                        } else k_soft<<<grid, 256, 0, s>>>(syncs, out, words);
                    }
                    cudaEventRecord(e1, s);
                    cudaEventSynchronize(e1);
                    float ms = 0;
                    cudaEventElapsedTime(&ms, e0, e1);
                    if (ms < best) best = ms;
                }
                printf("grid %4d CTAs, %d barriers/kernel, %-28s: %.2f us per kernel (chain of %d)\n", grid, syncs,
                       mode == 0 ? "plain launch" : mode == 1 ? "cooperative + grid.sync" : "plain + arrive/epoch barrier", best * 1e3f / chain, chain);
            }
        }
    }
    printf("last error: %s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
