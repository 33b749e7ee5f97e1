// Upper bound for a chain of DEPENDENT weight-streaming kernels (a decode step): every kernel streams `bytes` of fresh
// weights through per-warp cp.async.bulk rings, but may only start consuming after the previous kernel has finished
// (it reads a token the predecessor wrote).  With programmatic dependent launch and <= half an SM of resources per CTA the
// next kernel's CTAs become resident early and fill their rings BEFORE griddepcontrol.wait, so HBM keeps streaming across
// the kernel boundary.  Reports us / launch and TB/s for: plain stream order, PDL, PDL with a full-SM footprint (no
// co-residency), and a decode-shaped sequence (Q|K|V 25.5 MB, attention stub, O 8.5, gate|up 45.6, down 22.8) x 32.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o pdlchain pdlchain.cu && ./pdlchain
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile("{\n .reg .pred p;\n W: mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n @p bra D;\n bra W;\n D:\n}" ::"r"(bar), "r"(parity) : "memory");
}

constexpr int WARPS = 8, STAGES = 3;

// flags: 1 = call launch_dependents at the top, 2 = griddepcontrol.wait (else plain), 4 = consume (LDS) the data
__global__ void __launch_bounds__(WARPS * 32) k_stream(const uint8_t* __restrict__ src, size_t bytes, int stage, int flags,
                                                       const float* __restrict__ token_in, float* __restrict__ token_out, int epi_clks) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t bars[WARPS * STAGES];
    __shared__ float s_tok;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int gw = blockIdx.x * WARPS + warp, total_w = gridDim.x * WARPS;
    if (tid == 0) {
        for (int i = 0; i < WARPS * STAGES; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bars[i])));
        asm volatile("fence.mbarrier_init.release.cluster;");
    }
    __syncthreads();
    if (flags & 1) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    // this warp's contiguous byte range, in `stage`-byte copies
    const size_t n_all = bytes / stage;
    const size_t c0 = n_all * gw / total_w, c1 = n_all * (gw + 1) / total_w;
    const int n = (int)(c1 - c0);
    const uint8_t* base = src + c0 * (size_t)stage;
    uint8_t* ring = smem + (size_t)warp * STAGES * stage;
    int issued = 0;
    for (; issued < STAGES && issued < n; ++issued) {
        if (lane == 0) {
            const uint32_t b = smem_u32(&bars[warp * STAGES + issued]);
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"((uint32_t)stage) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                             smem_u32(ring + (size_t)issued * stage)), "l"(base + (size_t)issued * stage), "r"((uint32_t)stage), "r"(b) : "memory");
        }
    }
    if (flags & 2) asm volatile("griddepcontrol.wait;" ::: "memory");
    // "activation staging": a dependent global read + block barrier
    if (tid == 0) s_tok = token_in ? __ldcg(token_in) : 0.f;
    __syncthreads();
    uint32_t ph = 0, acc = __float_as_uint(s_tok);
    int st = 0;
    for (int i = 0; i < n; ++i) {
        mbar_wait(smem_u32(&bars[warp * STAGES + st]), (ph >> st) & 1u);
        ph ^= 1u << st;
        if (flags & 4) {
            const uint8_t* p = ring + (size_t)st * stage;
            for (int o = lane * 16; o < stage; o += 512) {
                const uint4 v = *reinterpret_cast<const uint4*>(p + o);
                acc += v.x ^ v.y ^ v.z ^ v.w;
            }
        }
        __syncwarp();
        if (issued < n) {
            if (lane == 0) {
                const uint32_t b = smem_u32(&bars[warp * STAGES + st]);
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"((uint32_t)stage) : "memory");
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                                 smem_u32(ring + (size_t)st * stage)), "l"(base + (size_t)issued * stage), "r"((uint32_t)stage), "r"(b) : "memory");
            }
            ++issued;
        }
        st = (st + 1 == STAGES) ? 0 : st + 1;
    }
    __syncthreads();
    if (epi_clks > 0) { const long long t0 = clock64(); while (clock64() - t0 < epi_clks) {} }
    if (tid == 0 && token_out) atomicAdd(token_out, __uint_as_float(acc & 0x007fffffu) * 1e-30f + 1.0f);
}

struct Step { size_t bytes; };

static float run_graph(const std::vector<Step>& steps, const uint8_t* wts, size_t wts_bytes, int stage, int smem_bytes, bool pdl,
                       bool early, int grid, float* tok, int reps, int epi_clks) {
    cudaStream_t s; CK(cudaStreamCreate(&s));
    CK(cudaFuncSetAttribute(k_stream, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    cudaGraph_t g; cudaGraphExec_t ge;
    CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    size_t off = 0;
    int idx = 0;
    for (const Step& st : steps) {
        if (off + st.bytes > wts_bytes) off = 0;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(grid); cfg.blockDim = dim3(WARPS * 32); cfg.dynamicSmemBytes = smem_bytes; cfg.stream = s;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
        const int flags = (pdl && early ? 1 : 0) | (pdl ? 2 : 0) | 4;
        CK(cudaLaunchKernelEx(&cfg, k_stream, wts + off, st.bytes, stage, flags, (const float*)(tok + (idx & 1)), tok + ((idx + 1) & 1), epi_clks));
        off += (st.bytes + 4095) / 4096 * 4096;
        ++idx;
    }
    CK(cudaStreamEndCapture(s, &g));
    CK(cudaGraphInstantiate(&ge, g, 0));
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    CK(cudaGraphLaunch(ge, s)); CK(cudaStreamSynchronize(s));
    CK(cudaEventRecord(a, s));
    for (int r = 0; r < reps; ++r) CK(cudaGraphLaunch(ge, s));
    CK(cudaEventRecord(b, s)); CK(cudaEventSynchronize(b));
    float ms; cudaEventElapsedTime(&ms, a, b);
    cudaGraphExecDestroy(ge); cudaGraphDestroy(g); cudaStreamDestroy(s);
    return ms / reps;
}

int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    const int sms = p.multiProcessorCount;
    printf("%s SMs %d\n", p.name, sms);
    const size_t wts_bytes = (size_t)4 << 30;
    uint8_t* wts; CK(cudaMalloc(&wts, wts_bytes)); CK(cudaMemset(wts, 1, wts_bytes));
    float* tok; CK(cudaMalloc(&tok, 64)); CK(cudaMemset(tok, 0, 64));
    const int stage = 4096;
    const int ring = WARPS * STAGES * stage;     // 96 KB
    struct Mode { const char* name; bool pdl, early; int smem; };
    const Mode modes[] = {{"stream order (no PDL)", false, false, ring},
                          {"PDL, wait only (trigger at exit)", true, false, ring},
                          {"PDL + early trigger, 97 KB/CTA (2 kernels co-resident)", true, true, ring + 1024},
                          {"PDL + early trigger, 200 KB/CTA (no co-residency)", true, true, 200 * 1024}};
    for (int epi : {0, 2000}) {
        printf("---- epilogue spin %d clk\n", epi);
        for (size_t mb10 : {85, 228, 456, 989}) {
            const size_t bytes = mb10 * 100000;
            std::vector<Step> steps(128, Step{bytes});
            for (const Mode& m : modes) {
                const float ms = run_graph(steps, wts, wts_bytes, stage, m.smem, m.pdl, m.early, sms, tok, 5, epi);
                printf("%5.1f MB x128  %-58s : %6.2f us/launch  %.2f TB/s\n", bytes * 1e-6, m.name, ms * 1e3 / 128, bytes * 128 / (ms * 1e-3) * 1e-12);
            }
        }
        // decode-shaped: per layer Q|K|V, attention stub (tiny), O, gate|up, down
        std::vector<Step> dec;
        size_t total = 0;
        for (int l = 0; l < 32; ++l) for (size_t b : {25500000ul, 200000ul, 8500000ul, 45600000ul, 22800000ul}) { dec.push_back(Step{b}); total += b; }
        for (const Mode& m : modes) {
            const float ms = run_graph(dec, wts, wts_bytes, stage, m.smem, m.pdl, m.early, sms, tok, 5, epi);
            printf("decode-shaped 160 launches %.2f GB  %-58s : %7.1f us/step  %.2f TB/s\n", total * 1e-9, m.name, ms * 1e3, total / (ms * 1e-3) * 1e-12);
        }
    }
    return 0;
}
