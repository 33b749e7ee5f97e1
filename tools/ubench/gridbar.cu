// Cost of a grid-wide phase barrier for a persistent decode kernel (DESIGN.md 7.1): 296 co-resident CTAs x 320 threads,
// one arrival per CTA on a global counter, everyone spins until all have arrived.  NOT YET RUN (written after round 1's
// GPU budget was spent).   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o gridbar gridbar.cu && ./gridbar
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include <cooperative_groups.h>
namespace cg = cooperative_groups;

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_release_add(unsigned* p, unsigned v) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// mode 0: red.release + ld.acquire spin;  mode 1: same with nanosleep back-off;  mode 2: cooperative_groups grid.sync()
__global__ void k_bar(unsigned* counters, int iters, int mode, long long* out) {
    cg::grid_group grid = cg::this_grid();
    const unsigned G = gridDim.x;
    __syncthreads();
    long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
        if (mode == 2) {
            grid.sync();
        } else {
            __syncthreads();
            if (threadIdx.x == 0) {
                red_release_add(counters + it, 1u);
                unsigned ns = 20;
                while (ld_acquire(counters + it) < G) {
                    if (mode == 1) { __nanosleep(ns); if (ns < 200) ns += 20; }
                }
            }
            __syncthreads();
        }
    }
    long long t1 = clock64();
    if (threadIdx.x == 0 && blockIdx.x == 0) out[0] = (t1 - t0) / iters;
}

int main() {
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    const int iters = 2000;
    unsigned* counters;
    long long* out;
    cudaMalloc(&counters, iters * sizeof(unsigned));
    cudaMallocManaged(&out, 8);
    for (int ctas_per_sm : {1, 2}) for (int mode : {0, 1, 2}) {
        cudaMemset(counters, 0, iters * sizeof(unsigned));
        int grid = sms * ctas_per_sm, threads = 320, it = iters;
        void* args[] = {&counters, &it, &mode, &out};
        cudaError_t e = cudaLaunchCooperativeKernel((void*)k_bar, dim3(grid), dim3(threads), args, 0, 0);
        cudaError_t e2 = cudaDeviceSynchronize();
        printf("ctas/SM %d mode %d (%s): %lld clk per barrier  (%s / %s)\n", ctas_per_sm, mode,
               mode == 0 ? "red.release + ld.acquire spin" : mode == 1 ? "same + nanosleep" : "cg grid.sync", out[0], cudaGetErrorString(e), cudaGetErrorString(e2));
    }
    return 0;
}
