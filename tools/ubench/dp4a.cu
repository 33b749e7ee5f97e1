// Can the CUDA cores keep up with HBM on a batch-1 dequant-GEMV if the dot product runs on the integer dot-product
// instruction (IDP.4A) instead of HFMA2?  Round-2 calibration for csrc/gemv_i8.cu.
//   A: raw IDP.4A issue rate (warp-instr / clk / SM)
//   B: the 4-bit inner loop of gemv_i8 on shared-memory-resident data: per 8 weights 2 LOP3 + 4 IDP.4A (16-bit
//      activations split into a signed high and an unsigned low byte plane), weights as LDS.128 (TC layout: one column per
//      lane, 8 k per word), activations as broadcast LDS.128.  Reports 4-bit weights / clk / SM; HBM needs 45 at 6.5 TB/s.
//   C: the reference-style HFMA2 loop (4 LOP3 + 1 SHF + 4 HADD2/HFMA2 + 4 HFMA2 per 8 weights) for comparison.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o dp4a dp4a.cu && ./dp4a
#include <cstdio>
#include <cstdint>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

__device__ __forceinline__ int dp4a_us(uint32_t a, uint32_t b, int c) {   // a unsigned bytes, b signed bytes
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
__device__ __forceinline__ int dp4a_uu(uint32_t a, uint32_t b, int c) {
    int d;
    asm("dp4a.u32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

__global__ void k_raw(int* out, int iters) {
    int acc[8];
    for (int i = 0; i < 8; ++i) acc[i] = threadIdx.x + i;
    uint32_t a = threadIdx.x * 0x01010101u, b = threadIdx.x * 0x03050709u;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = dp4a_us(a + i, b, acc[i]);
    }
    int s = 0;
    for (int i = 0; i < 8; ++i) s ^= acc[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// B: one warp = 64 columns (2 column blocks of the TC layout), slab = 32 k.
template <int NCOL>
__global__ void k_loop4(int* out, int slabs, int iters) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    // per warp: `slabs` slabs x NCOL blocks x 512 B of weights; shared activation planes 2 x 32 B per slab
    uint8_t* wbase = smem + (size_t)warp * slabs * NCOL * 512;
    uint8_t* abase = smem + (size_t)nw * slabs * NCOL * 512;
    for (int i = threadIdx.x; i < (nw * slabs * NCOL * 512 + slabs * 64) / 4; i += blockDim.x)
        reinterpret_cast<uint32_t*>(smem)[i] = i * 2654435761u;
    __syncthreads();
    int acc[NCOL][4];
    for (int c = 0; c < NCOL; ++c) for (int i = 0; i < 4; ++i) acc[c][i] = 0;
    float tot[NCOL] = {};
    for (int it = 0; it < iters; ++it) {
        for (int s = 0; s < slabs; ++s) {
            const uint4* ap = reinterpret_cast<const uint4*>(abase + s * 64);
            const uint4 ah0 = ap[0], ah1 = ap[1], al0 = ap[2], al1 = ap[3];
            const uint32_t AH[8] = {ah0.x, ah0.y, ah0.z, ah0.w, ah1.x, ah1.y, ah1.z, ah1.w};
            const uint32_t AL[8] = {al0.x, al0.y, al0.z, al0.w, al1.x, al1.y, al1.z, al1.w};
#pragma unroll
            for (int c = 0; c < NCOL; ++c) {
                const uint4 w4 = *reinterpret_cast<const uint4*>(wbase + ((size_t)s * NCOL + c) * 512 + lane * 16);
                const uint32_t W[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint32_t lo = W[j] & 0x0f0f0f0fu, hi = W[j] & 0xf0f0f0f0u;
                    acc[c][0] = dp4a_us(lo, AH[2 * j], acc[c][0]);
                    acc[c][1] = dp4a_uu(lo, AL[2 * j], acc[c][1]);
                    acc[c][2] = dp4a_us(hi, AH[2 * j + 1], acc[c][2]);
                    acc[c][3] = dp4a_uu(hi, AL[2 * j + 1], acc[c][3]);
                }
            }
            if ((s & 3) == 3) {          // group end (128 k): integer -> fp32 with the group scale
#pragma unroll
                for (int c = 0; c < NCOL; ++c) {
                    const int lo = (acc[c][0] << 8) + acc[c][1], hi = (acc[c][2] << 8) + acc[c][3];
                    tot[c] += (float)(lo * 16 + hi) * 0.37f;
                    acc[c][0] = acc[c][1] = acc[c][2] = acc[c][3] = 0;
                }
            }
        }
    }
    float r = 0;
    for (int c = 0; c < NCOL; ++c) r += tot[c];
    out[blockIdx.x * blockDim.x + threadIdx.x] = (int)r;
}

// C: HFMA2 loop, 2 columns per lane
__global__ void k_loop_h(int* out, int slabs, int iters) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    uint8_t* wbase = smem + (size_t)warp * slabs * 2 * 512;
    uint8_t* abase = smem + (size_t)nw * slabs * 2 * 512;
    for (int i = threadIdx.x; i < (nw * slabs * 2 * 512 + slabs * 64) / 4; i += blockDim.x)
        reinterpret_cast<uint32_t*>(smem)[i] = 0x3c003c00u;
    __syncthreads();
    half2 acc[2][2];
    for (int c = 0; c < 2; ++c) acc[c][0] = acc[c][1] = __float2half2_rn(0.f);
    float tot[2] = {};
    const half2 z1 = __float2half2_rn(-1032.f), m16 = __float2half2_rn(1.f / 16.f), z16 = __float2half2_rn(-72.f);
    for (int it = 0; it < iters; ++it) {
        for (int s = 0; s < slabs; ++s) {
            const uint4* ap = reinterpret_cast<const uint4*>(abase + s * 64);
            const uint4 a0 = ap[0], a1 = ap[1], a2 = ap[2], a3 = ap[3];
            const uint32_t A[16] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w, a2.x, a2.y, a2.z, a2.w, a3.x, a3.y, a3.z, a3.w};
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const uint4 w4 = *reinterpret_cast<const uint4*>(wbase + ((size_t)s * 2 + c) * 512 + lane * 16);
                const uint32_t W[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint32_t x = W[j], y = x >> 8;
                    uint32_t q0 = (x & 0x000f000fu) | 0x64006400u, q1 = (x & 0x00f000f0u) | 0x64006400u;
                    uint32_t q2 = (y & 0x000f000fu) | 0x64006400u, q3 = (y & 0x00f000f0u) | 0x64006400u;
                    const half2 h0 = __hadd2(*reinterpret_cast<half2*>(&q0), z1);
                    const half2 h1 = __hfma2(*reinterpret_cast<half2*>(&q1), m16, z16);
                    const half2 h2 = __hadd2(*reinterpret_cast<half2*>(&q2), z1);
                    const half2 h3 = __hfma2(*reinterpret_cast<half2*>(&q3), m16, z16);
                    acc[c][0] = __hfma2(h0, *reinterpret_cast<const half2*>(&A[4 * j + 0]), acc[c][0]);
                    acc[c][1] = __hfma2(h1, *reinterpret_cast<const half2*>(&A[4 * j + 1]), acc[c][1]);
                    acc[c][0] = __hfma2(h2, *reinterpret_cast<const half2*>(&A[4 * j + 2]), acc[c][0]);
                    acc[c][1] = __hfma2(h3, *reinterpret_cast<const half2*>(&A[4 * j + 3]), acc[c][1]);
                }
            }
            if ((s & 3) == 3) {
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const half2 t = __hadd2(acc[c][0], acc[c][1]);
                    tot[c] += (__low2float(t) + __high2float(t)) * 0.37f;
                    acc[c][0] = acc[c][1] = __float2half2_rn(0.f);
                }
            }
        }
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = (int)(tot[0] + tot[1]);
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
    int* out; cudaMalloc(&out, sms * 2048 * 4);
    const int iters = 4096;
    for (int warps : {4, 8, 16, 32}) {
        float ms = time_ms([&] { k_raw<<<sms, warps * 32>>>(out, iters); });
        printf("A raw IDP.4A  warps/SM %2d : %.3f warp-instr/clk/SM\n", warps, (double)iters * 8 * warps / (ms * 1e-3 * ghz * 1e9));
    }
    const int slabs = 8;
    for (int ctas : {1, 2}) for (int warps : {4, 8, 16}) {
        if (ctas * warps > 32) continue;
        {
            size_t sm = (size_t)warps * slabs * 2 * 512 + slabs * 64;
            cudaFuncSetAttribute(k_loop4<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
            float ms = time_ms([&] { k_loop4<2><<<sms * ctas, warps * 32, sm>>>(out, slabs, 512); });
            double w = 512.0 * slabs * 2 * 1024 * warps * ctas;
            printf("B dp4a loop 2 col/lane  ctas/SM %d warps/CTA %2d : %.1f weights/clk/SM  (%s)\n", ctas, warps, w / (ms * 1e-3 * ghz * 1e9), cudaGetErrorString(cudaGetLastError()));
        }
        {
            size_t sm = (size_t)warps * slabs * 4 * 512 + slabs * 64;
            cudaFuncSetAttribute(k_loop4<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
            float ms = time_ms([&] { k_loop4<4><<<sms * ctas, warps * 32, sm>>>(out, slabs, 512); });
            double w = 512.0 * slabs * 4 * 1024 * warps * ctas;
            printf("B dp4a loop 4 col/lane  ctas/SM %d warps/CTA %2d : %.1f weights/clk/SM  (%s)\n", ctas, warps, w / (ms * 1e-3 * ghz * 1e9), cudaGetErrorString(cudaGetLastError()));
        }
        {
            size_t sm = (size_t)warps * slabs * 2 * 512 + slabs * 64;
            cudaFuncSetAttribute(k_loop_h, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
            float ms = time_ms([&] { k_loop_h<<<sms * ctas, warps * 32, sm>>>(out, slabs, 512); });
            double w = 512.0 * slabs * 2 * 1024 * warps * ctas;
            printf("C hfma2 loop 2 col/lane ctas/SM %d warps/CTA %2d : %.1f weights/clk/SM  (%s)\n", ctas, warps, w / (ms * 1e-3 * ghz * 1e9), cudaGetErrorString(cudaGetLastError()));
        }
    }
    return 0;
}
