// Pipe-throughput calibration: legacy mma.sync (HMMA.16816.F32), LOP3, HADD2, LDS.128.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o pipes pipes.cu && ./pipes
#include <cstdio>
#include <cstdint>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

__global__ void k_hmma(float* out, int iters, int nacc) {
    float c[8][4];
    for (int i = 0; i < 8; ++i) for (int j = 0; j < 4; ++j) c[i][j] = 0.f;
    uint32_t a0 = threadIdx.x, a1 = a0 * 3, a2 = a0 * 5, a3 = a0 * 7, b0 = a0 * 11, b1 = a0 * 13;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (i < nacc)
            asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                : "+f"(c[i][0]), "+f"(c[i][1]), "+f"(c[i][2]), "+f"(c[i][3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
        }
    }
    float s = 0; for (int i = 0; i < 8; ++i) for (int j = 0; j < 4; ++j) s += c[i][j];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void k_alu(uint32_t* out, int iters) {
    uint32_t x[8];
    for (int i = 0; i < 8; ++i) x[i] = threadIdx.x * (i + 1);
    uint32_t m = 0x00f000f0u + (threadIdx.x & 1), g = 0x54005400u;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            uint32_t r;
            asm volatile("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(r) : "r"(x[i]), "r"(m), "r"(g));
            asm volatile("add.rn.f16x2 %0, %1, %2;" : "=r"(x[i]) : "r"(r), "r"(g));
        }
    }
    uint32_t s = 0; for (int i = 0; i < 8; ++i) s ^= x[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void k_mix(float* out, int iters) {   // per iteration: 8 (lop3 + shift) + 2 HMMA  ~ our 4-bit slab mix
    float c[2][4] = {};
    uint32_t x[4];
    for (int i = 0; i < 4; ++i) x[i] = threadIdx.x * (i + 1);
    uint32_t m = 0x00f000f0u, g = 0x54005400u, b0 = threadIdx.x, b1 = b0 * 3;
    for (int it = 0; it < iters; ++it) {
        uint32_t A[8];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            asm volatile("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(A[2 * i]) : "r"(x[i] << 4), "r"(m), "r"(g));
            asm volatile("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(A[2 * i + 1]) : "r"(x[i] >> 4), "r"(m), "r"(g));
            x[i] += A[2 * i];
        }
#pragma unroll
        for (int i = 0; i < 2; ++i)
            asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                : "+f"(c[i][0]), "+f"(c[i][1]), "+f"(c[i][2]), "+f"(c[i][3]) : "r"(A[4 * i]), "r"(A[4 * i + 1]), "r"(A[4 * i + 2]), "r"(A[4 * i + 3]), "r"(b0), "r"(b1));
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = c[0][0] + c[1][1] + c[0][2] + c[1][3];
}

template <typename F> float time_ms(F f) {
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    f(); cudaDeviceSynchronize();
    cudaEventRecord(a); f(); cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b); return ms;
}

int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    int sms = p.multiProcessorCount; double ghz = p.clockRate * 1e-6;
    printf("%s  SMs %d  clock %.3f GHz\n", p.name, sms, ghz);
    float* out; cudaMalloc(&out, sms * 8 * 1024 * 4);
    const int iters = 4096;
    for (int warps : {4, 8, 16, 32}) for (int nacc : {1, 2, 4, 8}) {
        float ms = time_ms([&] { k_hmma<<<sms, warps * 32>>>(out, iters, nacc); });
        double hmma_per_clk_sm = (double)iters * nacc * warps / (ms * 1e-3 * ghz * 1e9);
        printf("HMMA warps/SM %2d indep acc %d : %.3f HMMA/clk/SM  (%.0f dense-equivalent TFLOP/s)\n", warps, nacc, hmma_per_clk_sm,
               hmma_per_clk_sm * 4096 * sms * ghz * 1e-3);
    }
    for (int warps : {8, 16, 32}) {
        float ms = time_ms([&] { k_alu<<<sms, warps * 32>>>((uint32_t*)out, iters); });
        printf("LOP3+HADD2 pairs warps/SM %2d : %.3f warp-instr/clk/SM\n", warps, (double)iters * 16 * warps / (ms * 1e-3 * ghz * 1e9));
        ms = time_ms([&] { k_mix<<<sms, warps * 32>>>(out, iters); });
        printf("mix (8 lop3 + 8 shf + 4 add + 2 HMMA) warps/SM %2d : %.3f iterations/clk/SM -> %.1f weights/clk/SM\n", warps,
               (double)iters * warps / (ms * 1e-3 * ghz * 1e9), (double)iters * warps * 512 / (ms * 1e-3 * ghz * 1e9));
    }
    return 0;
}
