// Shared host/device helpers for libexl2b200 (sm_90a).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>

#include "../../include/exl2_b200.h"
#include "layout.h"

namespace exl2b {

// ---- error plumbing -------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launch_count;

#define EXL2B_CUDA(call)                                                                              \
    do {                                                                                              \
        cudaError_t _e = (call);                                                                      \
        if (_e != cudaSuccess) {                                                                      \
            exl2b::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return -1;                                                                                \
        }                                                                                             \
    } while (0)

#define EXL2B_REQUIRE(cond, ...)              \
    do {                                      \
        if (!(cond)) {                        \
            exl2b::set_error(__VA_ARGS__);    \
            return -2;                        \
        }                                     \
    } while (0)

// Launch with Programmatic Dependent Launch enabled: the kernel may start while its predecessor in the stream is
// still draining; it must call griddep_wait() before touching anything the predecessor writes.
// EXL2B_NO_PDL=1 (all kernels) or a list of kernel families (i8, tc, attn, small): plain stream-ordered launches (diagnostics)
inline bool pdl_disabled(const char* family) {
    static const char* e = getenv("EXL2B_NO_PDL");
    if (!e) return false;
    if (e[0] == '1' || e[0] == '\0') return true;
    return strstr(e, family) != nullptr;
}
inline bool slot_holders_disabled() {          // EXL2B_NO_HOLDERS=1: grids of working CTAs only (diagnostics)
    static const bool off = getenv("EXL2B_NO_HOLDERS") != nullptr;
    return off;
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_f(const char* family, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_disabled(family) ? 0 : 1;
    g_launch_count.fetch_add(1, std::memory_order_relaxed);
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_disabled("small") ? 0 : 1;
    g_launch_count.fetch_add(1, std::memory_order_relaxed);
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

int device_sm_count(int device);

// ---- slot holders -----------------------------------------------------------------------------------------------
// A launch whose grid has more CTAs than it has work for pads the grid to one CTA per SM: CTAs with blockIdx.x >= busy
// hold their SM slot (slot_hold) until every working CTA has left (slot_release), so that no SM runs two CTAs of one launch
// while another runs none (gemv_i8.cu).  The counter resets itself when the last CTA of the grid leaves.  Each kernel keeps
// a ring of 127 such counters per device, so a counter is reused only after 127 launches of that kernel.
struct SlotCounters {
    unsigned int* dev[64] = {};
    std::atomic<unsigned> seq{0};
};
inline int next_slot_counter(SlotCounters& s, int device, unsigned int** cnt) {
    if (!s.dev[device]) {
        EXL2B_CUDA(cudaMalloc(&s.dev[device], 128 * sizeof(unsigned int)));
        EXL2B_CUDA(cudaMemset(s.dev[device], 0, 128 * sizeof(unsigned int)));
    }
    *cnt = s.dev[device] + (s.seq.fetch_add(1) % 127u);
    return 0;
}

// ---- device-side PTX wrappers -----------------------------------------------------------------------------------
#if defined(__CUDACC__)

// one thread per CTA: count this CTA out of the launch
__device__ __forceinline__ void slot_release(unsigned int* cnt) {
    if (atomicAdd(cnt, 1u) == gridDim.x - 1u) *reinterpret_cast<volatile unsigned int*>(cnt) = 0u;
}
// one thread of a slot-holder CTA: wait for the `busy` working CTAs, then leave with them
__device__ __forceinline__ void slot_hold(unsigned int* cnt, int busy) {
    while (*reinterpret_cast<volatile unsigned int*>(cnt) < (unsigned)busy) __nanosleep(200);
    slot_release(cnt);
}

__device__ __forceinline__ unsigned long long globaltimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// optional phase stamps of a kernel whose params carry `dbg` / `dbg_cta` (exl2b_debug_set): stamp i of thread 0 of CTA dbg_cta;
// stamp 0 also lowers dbg[6] to the earliest start over the grid (the kernel raises dbg[7] to the latest end itself)
#define EXL2B_STAMP(P, i)                                                                                   \
    do {                                                                                                    \
        if ((P).dbg) {                                                                                      \
            if (blockIdx.x == (P).dbg_cta && threadIdx.x == 0) (P).dbg[i] = exl2b::globaltimer();         \
            if ((i) == 0 && threadIdx.x == 0) atomicMin((P).dbg + 6, exl2b::globaltimer());                \
        }                                                                                                   \
    } while (0)

// integer dot product of four byte pairs plus c.  a: 4 unsigned bytes; b: 4 signed (us) or unsigned (uu) bytes
__device__ __forceinline__ int dp4a_us(uint32_t a, uint32_t b, int c) {
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
__device__ __forceinline__ int dp4a_uu(uint32_t a, uint32_t b, int c) {
    int d;
    asm("dp4a.u32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
template <int BYTES>
__device__ __forceinline__ void cp_async_small(uint32_t dst, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(dst), "l"(src), "n"(BYTES) : "memory");
}

// ---- L2 eviction priority of data a decode step reads exactly once: the weights and the cached K/V rows.  A step streams
//      ~3.3 GB of them through the 50 MB L2; at normal priority they push out what every launch reuses (kernel code, launch
//      plans, norm weights, permutations, sin / cos, the rows one launch leaves for the next).  Loads and copies of such data
//      use the `_ef` variants below (evict-first); everything else keeps the unhinted helpers.
// Each variant makes its policy where it is used: a policy hoisted into a register and held across a loop costs the
// attention kernels, which sit at their 128-register cap, spills; made at each use (volatile, so it is not hoisted) it costs one
// instruction per copy and no register beyond the copy.
__device__ __forceinline__ uint64_t l2_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void cp_async16_ef(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "l"(l2_evict_first()) : "memory");
}
template <int BYTES>
__device__ __forceinline__ void cp_async_small_ef(uint32_t dst, const void* src) {
    asm volatile("cp.async.ca.shared.global.L2::cache_hint [%0], [%1], %2, %3;" ::"r"(dst), "l"(src), "n"(BYTES), "l"(l2_evict_first())
                 : "memory");
}
// read-only global load (the path __ldg takes), evict-first; T: uint8_t, uint16_t, uint32_t or uint4
template <typename T>
__device__ __forceinline__ T ldg_ef(const T* p) {
    const uint64_t pol = l2_evict_first();
    if constexpr (sizeof(T) == 16) {
        uint4 v;
        asm("ld.global.nc.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
            : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p), "l"(pol));
        return v;
    } else if constexpr (sizeof(T) == 4) {
        uint32_t v;
        asm("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
        return (T)v;
    } else if constexpr (sizeof(T) == 2) {
        unsigned short v;
        asm("ld.global.nc.L2::cache_hint.u16 %0, [%1], %2;" : "=h"(v) : "l"(p), "l"(pol));
        return (T)v;
    } else {
        static_assert(sizeof(T) == 1, "ldg_ef: 1, 2, 4 or 16 bytes");
        unsigned short v;
        asm("ld.global.nc.L2::cache_hint.u8 %0, [%1], %2;" : "=h"(v) : "l"(p), "l"(pol));
        return (T)v;
    }
}

__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t"
        "}" ::"r"(bar),
        "r"(parity)
        : "memory");
}
// TMA 1-D bulk copy global -> shared, completion on an mbarrier (SASS: UBLKCP).  16-byte aligned, size % 16 == 0.
__device__ __forceinline__ void bulk_copy_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
// the same, evict-first (l2_evict_first)
__device__ __forceinline__ void bulk_copy_g2s_ef(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(dst_smem),
                 "l"(src), "r"(bytes), "r"(bar), "l"(l2_evict_first())
                 : "memory");
}

// bulk prefetch of a global range into L2, evict-first (no shared memory, no completion to wait for).  16-byte aligned,
// size % 16 == 0.
__device__ __forceinline__ void bulk_prefetch_l2_ef(const void* src, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global.L2::cache_hint [%0], %1, %2;" ::"l"(src), "r"(bytes), "l"(l2_evict_first()) : "memory");
}

// D(16x8, f32) += A(16x16, f16, row) * B(16x8, f16, col)
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint2 lds64(uint32_t addr) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds_u16(uint32_t addr) {
    unsigned short v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ void stu128(uint32_t addr, uint4 v) {
    asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
// orders this thread's earlier generic-proxy shared-memory accesses before later async-proxy (bulk copy) writes
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// act(x) of act_mul (cuda/q_mlp_activation.cuh:54-130), shared by act_mul_kernel and the LoRA gate|up epilogue (lora.cu)
__device__ __forceinline__ half2 silu2(half2 x) {
    half2 one = __float2half2_rn(1.0f);
    half2 e = h2exp(__hneg2(x));
    half2 r = h2rcp(__hadd2(one, e));
    return __hmul2(x, r);
}
__device__ __forceinline__ half gelu1(half x) {
    float xf = __half2float(x);
    const float c = 0.797884560803f;
    float t = c * (xf + 0.044715f * xf * xf * xf), th;
    asm("tanh.approx.f32 %0, %1;" : "=f"(th) : "f"(t));
    xf = 0.5f * xf * (1.0 + th);
    return __float2half_rn(xf);
}
#endif

}  // namespace exl2b
