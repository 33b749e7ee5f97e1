// How fast can an SM pull HBM through per-warp cp.async.bulk rings?  Same fetch pattern as gemm_tc_kernel (every warp
// streams its own contiguous region in `stage` byte copies, `stages` in flight), but the consumer only waits and re-arms.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o bulkfetch bulkfetch.cu && ./bulkfetch
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile("{\n .reg .pred p;\n W: mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n @p bra D;\n bra W;\n D:\n}" ::"r"(bar), "r"(parity) : "memory");
}

// mode 0: every warp its own stream; mode 1: one thread per CTA issues copies of warps*stage bytes
__global__ void k_fetch(const uint8_t* src, size_t bytes_per_cta, int stage, int stages, int mode, int touch, unsigned* sink) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t bars[64];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nw = blockDim.x >> 5;
    const int streams = mode == 0 ? nw : 1;
    const int my = mode == 0 ? warp : 0;
    const size_t cs = mode == 0 ? (size_t)stage : (size_t)stage * nw;          // bytes per copy
    if (tid == 0) {
        for (int i = 0; i < streams * stages; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bars[i])));
        asm volatile("fence.mbarrier_init.release.cluster;");
    }
    __syncthreads();
    const size_t per_stream = bytes_per_cta / streams;
    const uint8_t* base = src + (size_t)blockIdx.x * bytes_per_cta + (size_t)my * per_stream;
    const int n = (int)(per_stream / cs);
    const bool issuer = (mode == 0) ? (lane == 0) : (tid == 0);
    const bool waiter = (mode == 0) ? true : true;
    uint32_t ph = 0, acc = 0;
    int issued = 0;
    for (; issued < stages && issued < n; ++issued) {
        if (issuer) {
            const uint32_t b = smem_u32(&bars[my * stages + issued]);
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"((uint32_t)cs) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                             smem_u32(smem + ((size_t)my * stages + issued) * cs)), "l"(base + (size_t)issued * cs), "r"((uint32_t)cs), "r"(b) : "memory");
        }
    }
    int st = 0;
    for (int i = 0; i < n; ++i) {
        if (waiter) mbar_wait(smem_u32(&bars[my * stages + st]), (ph >> st) & 1u);
        ph ^= 1u << st;
        if (touch) {
            const uint8_t* p = smem + ((size_t)my * stages + st) * cs + (mode == 0 ? 0 : (size_t)warp * stage);
            for (int o = lane * 16; o < stage; o += 512) {
                const uint4 v = *reinterpret_cast<const uint4*>(p + o);
                acc += v.x ^ v.y ^ v.z ^ v.w;
            }
        }
        if (mode == 1) __syncthreads();
        if (issued < n) {
            if (issuer) {
                const uint32_t b = smem_u32(&bars[my * stages + st]);
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"((uint32_t)cs) : "memory");
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                                 smem_u32(smem + ((size_t)my * stages + st) * cs)), "l"(base + (size_t)issued * cs), "r"((uint32_t)cs), "r"(b) : "memory");
            }
            ++issued;
        }
        st = (st + 1 == stages) ? 0 : st + 1;
    }
    if (acc == 0x12345678u) sink[0] = acc;
}

int main() {
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    const size_t total = (size_t)2 << 30;
    uint8_t* src;
    unsigned* sink;
    cudaMalloc(&src, total);
    cudaMalloc(&sink, 4);
    cudaMemset(src, 1, total);
    cudaFuncSetAttribute(k_fetch, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    printf("sms %d\n", sms);
    const int cfgs[][6] = {   // ctas/sm, warps, stage, stages, mode, touch
        {2, 8, 2560, 4, 0, 0}, {2, 8, 2560, 4, 0, 1}, {2, 8, 2048, 4, 0, 1}, {2, 8, 4096, 3, 0, 1}, {2, 8, 1024, 4, 0, 1},
        {1, 8, 2560, 4, 0, 1}, {1, 16, 2560, 4, 0, 1}, {2, 8, 2560, 2, 0, 1}, {2, 8, 2560, 3, 0, 1},
        {2, 8, 2560, 4, 1, 1}, {2, 8, 2560, 2, 1, 1}, {1, 8, 4096, 4, 1, 1}, {2, 4, 4096, 4, 0, 1}, {2, 8, 8192, 2, 0, 1},
    };
    for (auto& c : cfgs) {
        const int grid = sms * c[0], warps = c[1], stage = c[2], stages = c[3], mode = c[4], touch = c[5];
        size_t per_cta = total / grid;
        const size_t q = (size_t)warps * stage * 8;
        per_cta = per_cta / q * q;
        if (per_cta > (size_t)64 << 20) per_cta = ((size_t)64 << 20) / q * q;
        const size_t smem = (size_t)warps * stage * stages;
        for (int rep = 0; rep < 2; ++rep) {
            cudaEventRecord(e0);
            k_fetch<<<grid, warps * 32, smem>>>(src, per_cta, stage, stages, mode, touch, sink);
            cudaEventRecord(e1);
            cudaEventSynchronize(e1);
        }
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        cudaError_t err = cudaGetLastError();
        printf("ctas/sm %d warps %2d stage %5d stages %d mode %d touch %d  smem %6zu  bytes %.2f GB  %.3f ms  %.0f GB/s  %s\n", c[0], warps, stage, stages, mode,
               touch, smem, per_cta * (double)grid / 1e9, ms, per_cta * (double)grid / ms / 1e6, err == cudaSuccess ? "" : cudaGetErrorString(err));
    }
    return 0;
}
