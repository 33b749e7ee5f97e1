// gemv_i8_kernel -- the batch-1 (decode) dequant-GEMV of libexl2b200, HBM-bound by design.
// Replaces, for one input row, gemm_half_q_half_kernel / gemm_half_q_half_gptq_kernel (exllamav2_ext/cuda/q_gemm_kernel.cuh:
// 140-565, q_gemm_kernel_gptq.cuh:60-225) together with the kernels the reference runs in front of them (rms_norm_kernel,
// cuda/rms_norm.cu:55-143; act_mul_kernel, cuda/q_mlp_activation.cuh:54-100), which here are the kernel's PROLOGUE.
//
// Why integers: the reference's recipe (unpack to fp16, HFMA2) spends several CUDA-core instructions per weight, while the
// integer dot-product instruction (IDP.4A) consumes four packed fields per instruction (tools/ubench/dp4a.cu measures both
// loops on the GPU at hand).  So the row is quantised ONCE per launch to 16-bit integers per 128-k
// block with a power-of-two scale (signed high byte plane + unsigned low byte plane; values within 16x of the block
// maximum are exact, the rest carry |error| <= 2^-15 of the block maximum), packed weight fields are fed to dp4a without
// being expanded ((w & 0x0f0f0f0f) and (w & 0xf0f0f0f0) ARE four byte operands), integer sums are exact, and one fp32
// multiply per (column, group) applies weight scale x row scale.  Zero points come out as  -zero * sum(row block).
//
// Why this shape: a decode step is a chain of ~160 DEPENDENT launches of 8-45 MB each; what bounds it is the serial latency
// of every launch (measured with the phase stamps below), not instruction throughput.  So:
//   * one CTA per SM, 16 warps, <= 111 KB of shared memory: TWO consecutive launches are co-resident.  A CTA's first action is
//     griddepcontrol.launch_dependents and every warp requests its first weight stages BEFORE griddepcontrol.wait, so while
//     launch N computes, launch N+1 is already filling its arenas and HBM keeps streaming across the kernel boundary
//     (tools/ubench/pdlchain.cu compares a decode-shaped chain of dependent launches with and without this overlap).
//   * every grid is EXACTLY one CTA per SM: CTAs without blocks are slot holders (see the kernel), so no SM ever runs two CTAs
//     of the same launch while another idles.
//   * a CTA owns WHOLE 32-column blocks (all of K), its 16 warps split the blocks' K range between them: split-K never leaves
//     the CTA (shared memory + one barrier), there is no workspace, no atomics, no fence, and summation order is fixed.
//   * everything positional (block -> CTA partition, every warp's stage list, who holds partial sums of which block) is a
//     launch PLAN built on the host once per matrix structure (I8Plan below): the device walks 16-byte descriptors.
//   * a warp streams its share of a block's bytes (layout.h: one contiguous stream per block) with cp.async.bulk into a
//     private byte arena (a ring of variable-size stages placed by the host) and never synchronises with another warp in the
//     main loop; per quantisation group one fp32 FMA with a scale from the matrix' dense scale table (QMatrix::wtab).  The
//     main loop issues no global load that it waits for: a group's scale row travels with the group's last stage (same bulk
//     copy barrier) and the stage list is read from a shared-memory window that the stage copies refill ahead of use.
//   * when the producer of the row scattered a copy in this matrix's stored-row order (I8Out::c_perm), the prologue reads the
//     row with one 16-byte load per thread instead of eight 2-byte gathers.
#include <string.h>

#include <algorithm>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "gemv_i8.cuh"

namespace exl2b {

constexpr int I8_MAX_WARPS = 16;
constexpr int I8_MAX_CTAS = 320;

struct I8Mat {
    const uint8_t* packed;
    const void* wtab;                 // dense scale table (QMatrix::wtab): EXL2 fp16[G][N], GPTQ uint32[G][N]
    const half* bias;
    half* c;
    half* c_perm;
    const uint16_t* out_invperm;
    int N, blk_base, clear;
};

// One stage of a warp's work = one bulk copy = up to 4 slabs of one 32-column block with one bit width, inside one
// quantisation group and one 128-k row block.  16 bytes, built ON THE HOST once per launch structure (I8Plan below):
//   x = byte offset of the stage inside its matrix' packed buffer
//   y = element index of lane 0's entry in the matrix' scale table (group * N + first column of the block)
//   z = ks | slabs << 11 | bits << 14 | flags << 18 | matrix << 22 | (bytes / 128) << 24
//   w = block index relative to the CTA's first block | (byte offset of the stage in the warp's arena / 128) << 16
//       | (stages to request once this one is consumed) << 24
// A warp's weight arena is a byte ring (not fixed slots): the host places every stage, records after which stage's consumption its
// space is free (that is the `request` count above), and the first stages -- everything that fits the arena, for small matrices the
// warp's WHOLE share -- are requested before the dependency wait.  Stage s completes on mbarrier s % I8_BARS, parity (s / I8_BARS) & 1.
// The same barrier covers two small copies that travel with stage s:
//   * for a DF_FLUSH stage, the 32-column scale row of its group (64 B of fp16, or 128 B of GPTQ scale | zero << 16) into slot
//     s % I8_BARS of the warp's scale ring.  At most I8_BARS stages are in flight, so stage s + I8_BARS (the next user of the
//     slot) is requested only after stage s has been consumed.
//   * descriptor s + I8_BARS into slot (s + I8_BARS) % I8_LWIN of the warp's list window.  Consuming stage s reads descriptor s
//     and requests stages up to s + I8_BARS, all of which arrived with stages <= s; the slot it overwrites held descriptor
//     s - I8_BARS, consumed before stage s could be requested.  Descriptors 0 .. I8_BARS - 1 are loaded before the first request.
constexpr uint32_t DF_FLUSH = 1, DF_BLOCK_DONE = 2, DF_GPTQ = 4;
constexpr int I8_BARS = 8;
constexpr int I8_LWIN = 2 * I8_BARS;

struct I8Params {
    I8Mat mat[I8_MAX_MATS];
    const uint4* plan_desc;           // stage descriptors, warp after warp, CTA after CTA
    const uint32_t* plan_first;       // [ctas * warps + 1] first descriptor of every warp | stages to request up front << 26
    const uint32_t* plan_cta;         // [ctas] first block | blocks << 16
    const uint32_t* plan_red;         // [blocks] bit w: warp w holds a partial sum of the block | the first such warp's partial slot << 16
    int num_mats, K, KS;
    const uint16_t* perm;             // stored row k' <- feature perm[k'], or NULL
    const half* x;
    const half* x2;
    const half* norm_w;
    float norm_eps;
    int mode, x_permuted;
    int norm_permuted;                // norm_w is already in stored-row order (I8Input::norm_wp)
    int l2_prefetch;                  // prefetch the part of a warp's share that does not fit its arena into L2 before the wait
    int arena;                        // bytes of a warp's weight arena
    int srow;                         // bytes of a scale ring slot: 64 (fp16 scale rows), 128 when a matrix is GPTQ
    int busy_ctas;                    // CTAs that own blocks; the rest of the grid only keeps its SM slot occupied (see the kernel)
    unsigned int* slot_cnt;           // CTAs of this launch that are done (self-resetting)
    unsigned long long* dbg;          // optional globaltimer stamps (exl2b_debug_set), NULL in production
    int dbg_cta;
    unsigned long long* dbg_rec;      // optional per-CTA records [cta][4]: start, dependency wait over, end, SM id
};

// dynamic shared-memory map of a CTA (byte offsets, every region 16-byte aligned) -- one definition for host and device
struct I8Smem {
    uint32_t act, asum, ascale, emit, scl, lst, total;
};
__host__ __device__ inline I8Smem i8_smem_map(int warps, int arena, int KS, int srow) {
    auto up = [](uint32_t x) { return (x + 15u) & ~15u; };
    I8Smem m;
    m.act = up((uint32_t)warps * (uint32_t)arena);                   // staged row: [KS][64 B]
    m.asum = up(m.act + (uint32_t)KS * 64u);                          // [KS] integer sum of a slab's row values
    m.ascale = up(m.asum + (uint32_t)KS * 4u);                        // [KS/4 + 1] scale of a 128-k block
    m.emit = up(m.ascale + (uint32_t)(KS / 4 + 1) * 4u);              // [warp][2][32] partial sums of split blocks
    m.scl = up(m.emit + (uint32_t)warps * 256u);                      // [warp][I8_BARS][srow] scale rows of the flush stages in flight
    m.lst = up(m.scl + (uint32_t)(warps * I8_BARS * srow));           // [warp][I8_LWIN] stage-list window (16-byte descriptors)
    m.total = up(m.lst + (uint32_t)(warps * I8_LWIN * 16));
    return m;
}

// ---- one slab (32 k) of the warp's 32-column block: integer dot products, one column per lane -------------------------------
// Staged row of a slab (64 B): XH[2j] / XH[2j+1] = high bytes of k = 8j + {0,4,1,5} / 8j + {2,6,3,7}; XL the low bytes.
// That is the byte order every plane's masked words have (layout.h pair_word / pair_slot): (w & 0x0f0f0f0f) / (w & 0xf0f0f0f0)
// of 4-bit word j meet XH[2j] / XH[2j+1]; field position i of 2-bit word w meets XH[4w + i]; bit position i of the 1-bit word
// meets XH[i]; 8-bit word w meets XH[w].  No operand is ever permuted.
template <int BITS>
__device__ __forceinline__ void consume_slab(uint32_t wb, uint32_t xs, int lane, int (&am)[4], int (&ae)[2]) {
    constexpr int Pm = plane_main(BITS), Pe = plane_extra(BITS);
    if constexpr (BITS == 4) {
        // the common case, in two halves of the slab so that only 8 row words are live at a time (64 registers per thread)
        const uint4 w4 = lds128(wb + lane * 16);
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            const uint4 xh = lds128(xs + hf * 16), xl = lds128(xs + 32 + hf * 16);
            const uint32_t wa = hf ? w4.z : w4.x, wc = hf ? w4.w : w4.y;
            const uint32_t lo0 = wa & 0x0f0f0f0fu, hi0 = wa & 0xf0f0f0f0u, lo1 = wc & 0x0f0f0f0fu, hi1 = wc & 0xf0f0f0f0u;
            am[0] = dp4a_us(lo0, xh.x, am[0]);
            am[1] = dp4a_uu(lo0, xl.x, am[1]);
            am[2] = dp4a_us(hi0, xh.y, am[2]);
            am[3] = dp4a_uu(hi0, xl.y, am[3]);
            am[0] = dp4a_us(lo1, xh.z, am[0]);
            am[1] = dp4a_uu(lo1, xl.z, am[1]);
            am[2] = dp4a_us(hi1, xh.w, am[2]);
            am[3] = dp4a_uu(hi1, xl.w, am[3]);
        }
        return;
    }
    uint32_t XH[8], XL[8];
    {
        const uint4 h0 = lds128(xs), h1 = lds128(xs + 16), l0 = lds128(xs + 32), l1 = lds128(xs + 48);
        XH[0] = h0.x; XH[1] = h0.y; XH[2] = h0.z; XH[3] = h0.w; XH[4] = h1.x; XH[5] = h1.y; XH[6] = h1.z; XH[7] = h1.w;
        XL[0] = l0.x; XL[1] = l0.y; XL[2] = l0.z; XL[3] = l0.w; XL[4] = l1.x; XL[5] = l1.y; XL[6] = l1.z; XL[7] = l1.w;
    }
    // ---- main plane
    if constexpr (Pm == 4) {
        const uint4 w4 = lds128(wb + lane * 16);
        const uint32_t W[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t lo = W[j] & 0x0f0f0f0fu, hi = W[j] & 0xf0f0f0f0u;      // hi carries a factor 16 (removed at the flush)
            am[0] = dp4a_us(lo, XH[2 * j], am[0]);
            am[1] = dp4a_uu(lo, XL[2 * j], am[1]);
            am[2] = dp4a_us(hi, XH[2 * j + 1], am[2]);
            am[3] = dp4a_uu(hi, XL[2 * j + 1], am[3]);
        }
    } else if constexpr (Pm == 8) {
        const uint4 a4 = lds128(wb + lane * 16), b4 = lds128(wb + 512 + lane * 16);
        const uint32_t W[8] = {a4.x, a4.y, a4.z, a4.w, b4.x, b4.y, b4.z, b4.w};
#pragma unroll
        for (int w = 0; w < 8; ++w) {
            am[0] = dp4a_us(W[w], XH[w], am[0]);
            am[1] = dp4a_uu(W[w], XL[w], am[1]);
        }
    } else {   // Pm == 2: field position i of word w meets operand word 4w + i
        const uint2 w2 = lds64(wb + lane * 8);
        const uint32_t W[2] = {w2.x, w2.y};
#pragma unroll
        for (int w = 0; w < 2; ++w)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const uint32_t t = (W[w] >> (2 * i)) & 0x03030303u;
                am[0] = dp4a_us(t, XH[4 * w + i], am[0]);
                am[1] = dp4a_uu(t, XL[4 * w + i], am[1]);
            }
    }
    // ---- extra plane (bits above the main plane), at byte 128 * Pm of the block
    if constexpr (Pe == 1) {   // one word: bit position i meets operand word i
        const uint32_t w = lds32(wb + 128 * Pm + lane * 4);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const uint32_t t = (w >> i) & 0x01010101u;
            ae[0] = dp4a_us(t, XH[i], ae[0]);
            ae[1] = dp4a_uu(t, XL[i], ae[1]);
        }
    } else if constexpr (Pe == 2) {
        const uint2 w2 = lds64(wb + 128 * Pm + lane * 8);
        const uint32_t W[2] = {w2.x, w2.y};
#pragma unroll
        for (int w = 0; w < 2; ++w)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const uint32_t t = (W[w] >> (2 * i)) & 0x03030303u;
                ae[0] = dp4a_us(t, XH[4 * w + i], ae[0]);
                ae[1] = dp4a_uu(t, XL[4 * w + i], ae[1]);
            }
    }
}

template <int BITS>
__device__ __forceinline__ int consume_stage(uint32_t slot, int n, uint32_t xs, uint32_t asum, int lane, int (&am)[4], int (&ae)[2]) {
    constexpr uint32_t bb = 128 * BITS;
    int S = 0;
    if constexpr (BITS == 4) {
        // the common case: the lane's weight words of slab s + 1 are loaded before the arithmetic of slab s (the shared-memory round
        // trip of the one non-broadcast load hides behind 16 dot products)
        uint4 w4 = lds128(slot + lane * 16);
#pragma unroll 1
        for (int s = 0; s < n; ++s) {
            const uint4 wn = lds128(slot + (s + 1 < n ? s + 1 : s) * bb + lane * 16);
            const uint32_t x = xs + s * 64;
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                const uint4 xh = lds128(x + hf * 16), xl = lds128(x + 32 + hf * 16);
                const uint32_t wa = hf ? w4.z : w4.x, wc = hf ? w4.w : w4.y;
                const uint32_t lo0 = wa & 0x0f0f0f0fu, hi0 = wa & 0xf0f0f0f0u, lo1 = wc & 0x0f0f0f0fu, hi1 = wc & 0xf0f0f0f0u;
                am[0] = dp4a_us(lo0, xh.x, am[0]);
                am[1] = dp4a_uu(lo0, xl.x, am[1]);
                am[2] = dp4a_us(hi0, xh.y, am[2]);
                am[3] = dp4a_uu(hi0, xl.y, am[3]);
                am[0] = dp4a_us(lo1, xh.z, am[0]);
                am[1] = dp4a_uu(lo1, xl.z, am[1]);
                am[2] = dp4a_us(hi1, xh.w, am[2]);
                am[3] = dp4a_uu(hi1, xl.w, am[3]);
            }
            S += (int)lds32(asum + s * 4);
            w4 = wn;
        }
        return S;
    }
#pragma unroll 1
    for (int s = 0; s < n; ++s) {
        consume_slab<BITS>(slot + s * bb, xs + s * 64, lane, am, ae);
        S += (int)lds32(asum + s * 4);
    }
    return S;
}

// One lane's output of block `blk`: what is added to it / where its copy in the consumer's row order goes is LOADED by out_pre
// (raw bits: nothing there waits for memory; the launch's tail calls it before the main loop and touches the values after it),
// the addresses are recomputed by finalize_block.
struct I8OutPre {
    uint32_t add;         // fp16 bits of bias[n] | fp16 bits of the old c[n] << 16   (0 where absent)
    uint32_t kp;          // index in the consumer's stored-row order (c_perm)
};
__device__ __forceinline__ int mat_of_block(const I8Params& P, int blk) {
    int mi = 0;
#pragma unroll
    for (int i = 1; i < I8_MAX_MATS; ++i)
        if (i < P.num_mats && blk >= P.mat[i].blk_base) mi = i;
    return mi;
}
__device__ __forceinline__ I8OutPre out_pre(const I8Params& P, int blk, int lane) {
    const I8Mat& m = P.mat[mat_of_block(P, blk)];
    const int n = (blk - m.blk_base) * 32 + lane;
    I8OutPre r = {0u, (uint32_t)n};
    if (n < m.N) {
        if (m.bias) r.add = __ldg(reinterpret_cast<const unsigned short*>(m.bias) + n);
        if (!m.clear) r.add |= (uint32_t)__ldcg(reinterpret_cast<const unsigned short*>(m.c) + n) << 16;
        if (m.c_perm && m.out_invperm) r.kp = __ldg(m.out_invperm + n);
    }
    return r;
}
__device__ __forceinline__ void finalize_block(const I8Params& P, int blk, int lane, const I8OutPre& pre, float v) {
    const I8Mat& m = P.mat[mat_of_block(P, blk)];
    const int n = (blk - m.blk_base) * 32 + lane;
    if (n < m.N) {
        v += __half2float(__ushort_as_half((unsigned short)(pre.add & 0xffffu)));          // bias first, then the old value
        v += __half2float(__ushort_as_half((unsigned short)(pre.add >> 16)));
        const half h = __float2half_rn(v);
        m.c[n] = h;
        if (m.c_perm) m.c_perm[pre.kp] = h;
    }
}

__device__ __forceinline__ half silu_h(half x) {        // cuda/q_mlp_activation.cuh:13-23, same fp16 op sequence
    const half e = hexp(__hneg(x));
    const half r = hrcp(__hadd(__float2half(1.0f), e));
    return __hmul(x, r);
}
__device__ __forceinline__ half2 silu_h2(half2 x) {     // the same op sequence on two values at once (packed fp16 instructions)
    const half2 e = h2exp(__hneg2(x));
    const half2 r = h2rcp(__hadd2(__float2half2_rn(1.0f), e));
    return __hmul2(x, r);
}
__device__ __forceinline__ half gelu_h(half x) {        // cuda/q_mlp_activation.cuh:37-47
    float xf = __half2float(x);
    const float t = 0.797884560803f * (xf + 0.044715f * xf * xf * xf);
    float th;
    asm("tanh.approx.f32 %0, %1;" : "=f"(th) : "f"(t));
    xf = 0.5f * xf * (1.0 + th);
    return __float2half_rn(xf);
}

// stamps of thread 0 of CTA dbg_cta: 0 start, 1 first stages requested, 2 dependency wait over, 3 row staged,
// 4 warp 0's main loop done, 5 all warps done, (6 = earliest CTA start, 7 = latest CTA end over the grid), 8 stage list in
// shared memory, 9 first stages and scales requested (EXL2B_STAMP)

// ---- the kernel -----------------------------------------------------------------------------------------------------------
template <int I8_WARPS>
__global__ void __launch_bounds__(I8_WARPS * 32, 2) gemv_i8_kernel(const __grid_constant__ I8Params P) {
    constexpr int I8_THREADS = I8_WARPS * 32;
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t bars[I8_WARPS * I8_BARS];
    __shared__ float s_red[I8_WARPS];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int KS = P.KS;
    EXL2B_STAMP(P, 0);
    if (P.dbg_rec && tid == 0 && blockIdx.x < 160) P.dbg_rec[blockIdx.x * 4] = globaltimer();
    if (tid < I8_WARPS * I8_BARS) mbar_init(smem_addr(&bars[tid]), 1);
    mbar_fence_init();
    __syncthreads();
    griddep_launch_dependents();          // the next launch may become resident (and prefetch ITS weights) right away

    // ---- slot holders.  The grid always has one CTA per SM.  With two launches co-resident per SM, every SM must host exactly
    //      ONE CTA of every launch of the chain: an SM that has none would offer two free slots to the next launch, which then
    //      runs two of its CTAs there at half speed each while another SM idles.  So CTAs without blocks stay resident until the CTAs with blocks are done, then leave with them.
    if ((int)blockIdx.x >= P.busy_ctas) {
        if (tid == 0) slot_hold(P.slot_cnt, P.busy_ctas);
        return;
    }

    // ---- this CTA's blocks and this warp's stage list, straight from the host-built plan (nothing here depends on the
    //      previous launch).
    const uint32_t cinfo = __ldg(P.plan_cta + blockIdx.x);
    const int blk0 = (int)(cinfo & 0xffffu), nb = (int)(cinfo >> 16);
    const uint32_t fw0 = __ldg(P.plan_first + blockIdx.x * I8_WARPS + warp), fw1 = __ldg(P.plan_first + blockIdx.x * I8_WARPS + warp + 1);
    const uint32_t f0 = fw0 & 0x3ffffffu, f1 = fw1 & 0x3ffffffu;
    const int nst = (int)(f1 - f0), n_pre = (int)(fw0 >> 26);
    const uint4* const list = P.plan_desc + f0;

    // shared-memory map: generic pointers for the prologue's stores, 32-bit shared-space addresses (`lds*`) for the main loop
    const I8Smem sm = i8_smem_map(I8_WARPS, P.arena, KS, P.srow);
    uint8_t* const act_g = smem + sm.act;
    int* const asum_s = reinterpret_cast<int*>(smem + sm.asum);
    float* const ascale_s = reinterpret_cast<float*>(smem + sm.ascale);
    float* const emit_base = reinterpret_cast<float*>(smem + sm.emit);
    uint32_t sbase;        // kept opaque: the compiler would otherwise re-derive every shared address from S2R in the loop
    asm volatile("mov.u32 %0, %1;" : "=r"(sbase) : "r"(smem_addr(smem)));
    const uint32_t ring = sbase + (uint32_t)warp * (uint32_t)P.arena;
    const uint32_t act = sbase + sm.act, asum = sbase + sm.asum, ascale = sbase + sm.ascale;
    const uint32_t sring = sbase + sm.scl + (uint32_t)(warp * I8_BARS * P.srow), lwin = sbase + sm.lst + (uint32_t)(warp * I8_LWIN * 16);
    uint32_t bar0;
    asm volatile("mov.u32 %0, %1;" : "=r"(bar0) : "r"(smem_addr(&bars[warp * I8_BARS])));

    // request stages [s0, s0 + cnt) into their places in the arena: lane j decodes and issues stage s0 + j (cnt <= I8_BARS), so
    // a batch of requests costs one descriptor decode, not one per stage.  `d` is lane j's descriptor (stage s0 + j).  With the
    // stage come its group's scale row (flush stages) and descriptor s + I8_BARS, on the same barrier (see DF_FLUSH above).
    // Weights and scale rows are read once per step: evict-first in L2.  The descriptor is not: every layer's launch of the same
    // structure walks the same plan.
    auto issue_stages = [&](int s0, int cnt, uint4 d) {
        if (lane < cnt) {
            const int s = s0 + lane;
            const uint32_t mi = (d.z >> 22) & 3u;
            const uint8_t* pk = mi == 0 ? P.mat[0].packed : (mi == 1 ? P.mat[1].packed : P.mat[2].packed);
            const uint8_t* wt = reinterpret_cast<const uint8_t*>(mi == 0 ? P.mat[0].wtab : (mi == 1 ? P.mat[1].wtab : P.mat[2].wtab));
            const uint32_t bytes = ((d.z >> 24) & 0xffu) << 7;
            const uint32_t esz = (d.z & (DF_GPTQ << 18)) ? 4u : 2u;
            const uint32_t sbytes = (d.z & (DF_FLUSH << 18)) ? 32u * esz : 0u;
            const bool lnext = s + I8_BARS < nst;
            const uint32_t slot = (uint32_t)s & (I8_BARS - 1);
            const uint32_t bar = bar0 + slot * 8u;
            mbar_arrive_expect_tx(bar, bytes + sbytes + (lnext ? 16u : 0u));
            bulk_copy_g2s_ef(ring + ((d.w >> 16) & 0xffu) * 128u, pk + d.x, bytes, bar);
            if (sbytes) bulk_copy_g2s_ef(sring + slot * (uint32_t)P.srow, wt + (size_t)d.y * esz, sbytes, bar);
            if (lnext) bulk_copy_g2s(lwin + ((uint32_t)(s + I8_BARS) & (I8_LWIN - 1)) * 16u, list + s + I8_BARS, 16u, bar);
        }
    };
    // descriptors 0 .. I8_BARS - 1 into the window; every later one arrives with the stage I8_BARS before it
    uint4 dfirst = make_uint4(0u, 0u, 0u, 0u);
    if (lane < I8_BARS && lane < nst) {
        dfirst = __ldg(list + lane);
        stu128(lwin + (uint32_t)lane * 16u, dfirst);
    }
    fence_proxy_async();                   // these window slots are later overwritten by bulk copies
    __syncwarp();
    EXL2B_STAMP(P, 8);
    issue_stages(0, n_pre, dfirst);
    int next_req = n_pre;
    // EXPERIMENT, off by default (EXL2B_I8_L2PF=1): pull the rest of the warp's share into L2 now (one bulk prefetch per stage),
    // while the previous launch is still computing.  Off because the 20-30 MB burst of the next launch competes with the
    // running launch's own refills.
    if (P.l2_prefetch)
        for (int s0 = n_pre; s0 < nst; s0 += 32) {
            const int s = s0 + lane;
            if (s < nst) {
                const uint4 d = __ldg(list + s);
                const uint32_t mi = (d.z >> 22) & 3u;
                const uint8_t* pk = mi == 0 ? P.mat[0].packed : (mi == 1 ? P.mat[1].packed : P.mat[2].packed);
                bulk_prefetch_l2_ef(pk + d.x, ((d.z >> 24) & 0xffu) << 7);
            }
        }
    EXL2B_STAMP(P, 9);

    // ---- static operands of the prologue, fetched before the dependency wait: permutation indices (when the row has to be
    //      gathered, or the norm weight has) and the norm weight of this thread's first octets
    const int n_oct = P.K >> 3;
    const bool gather_x = P.perm != nullptr && !P.x_permuted;
    constexpr int PF = 3;
    uint4 pv[PF], wv[PF];
#pragma unroll
    for (int r = 0; r < PF; ++r) {
        const int o = r * I8_THREADS + tid;
        pv[r] = make_uint4(0, 0, 0, 0);
        wv[r] = make_uint4(0, 0, 0, 0);
        if (o < n_oct) {
            if (P.perm && (gather_x || !P.norm_permuted)) pv[r] = __ldg(reinterpret_cast<const uint4*>(P.perm + o * 8));
            if (P.mode == I8_RMSNORM) {
                if (P.perm && !P.norm_permuted) {
                    const uint16_t* pi = reinterpret_cast<const uint16_t*>(&pv[r]);
                    uint16_t* wo = reinterpret_cast<uint16_t*>(&wv[r]);
#pragma unroll
                    for (int e = 0; e < 8; ++e) wo[e] = __half_as_ushort(__ldg(P.norm_w + pi[e]));
                } else {
                    wv[r] = __ldg(reinterpret_cast<const uint4*>(P.norm_w + o * 8));
                }
            }
        }
    }

    EXL2B_STAMP(P, 1);
    griddep_wait();                        // everything below may read what the previous launch wrote
    EXL2B_STAMP(P, 2);
    if (P.dbg_rec && tid == 0 && blockIdx.x < 160) P.dbg_rec[blockIdx.x * 4 + 1] = globaltimer();

    // ---- prologue: the row -> (optional RMSNorm weight / act*mul) -> 16-bit integers per 128-k block -> shared memory.
    //      Every CTA stages the whole row (its blocks span all of K); 1/rms is applied to the finished fp32 sums.
    float sumsq = 0.f;
    // A row that has to be gathered through q_perm is first copied into shared memory with coalesced 16-byte loads (into the
    // region that will hold the staged integers: same size) and gathered from there: one L2 round trip instead of eight
    // scattered 2-byte sector reads per thread.
    const bool two_in = (P.mode == I8_SILU_MUL || P.mode == I8_GELU_MUL);
    const bool smem_gather = gather_x && !two_in && n_oct <= PF * I8_THREADS;
    uint4 hg[PF];
    if (smem_gather) {
        for (int o = tid; o < n_oct; o += I8_THREADS)
            reinterpret_cast<uint4*>(act_g)[o] = __ldcg(reinterpret_cast<const uint4*>(P.x + o * 8));
        __syncthreads();
#pragma unroll
        for (int r = 0; r < PF; ++r) {
            const int o = r * I8_THREADS + tid;
            hg[r] = make_uint4(0, 0, 0, 0);
            if (o < n_oct) {
                const uint16_t* pi = reinterpret_cast<const uint16_t*>(&pv[r]);
                uint16_t* ho = reinterpret_cast<uint16_t*>(&hg[r]);
#pragma unroll
                for (int e = 0; e < 8; ++e) ho[e] = reinterpret_cast<const uint16_t*>(act_g)[pi[e]];
            }
        }
        __syncthreads();
    }
    auto stage_round = [&](int o, uint4 pidx, uint4 wreg, bool pre, uint4 hval) {
        const bool valid = o < n_oct;
        float f[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = 0.f;
        if (valid) {
            const uint16_t* pi = reinterpret_cast<const uint16_t*>(&pidx);
            half h[8], h2[8];
            const bool two = two_in;
            if (pre) {
                *reinterpret_cast<uint4*>(h) = hval;
            } else if (gather_x) {
#pragma unroll
                for (int e = 0; e < 8; ++e) h[e] = __ldcg(P.x + pi[e]);
                if (two) {
#pragma unroll
                    for (int e = 0; e < 8; ++e) h2[e] = __ldcg(P.x2 + pi[e]);
                }
            } else {
                const uint4 v = __ldcg(reinterpret_cast<const uint4*>(P.x + o * 8));
                *reinterpret_cast<uint4*>(h) = v;
                if (two) *reinterpret_cast<uint4*>(h2) = __ldcg(reinterpret_cast<const uint4*>(P.x2 + o * 8));
            }
            if (P.mode == I8_RMSNORM) {
                const half* wh = reinterpret_cast<const half*>(&wreg);
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const float xf = __half2float(h[e]);
                    sumsq = fmaf(xf, xf, sumsq);
                    f[e] = xf * __half2float(wh[e]);
                }
            } else if (P.mode == I8_SILU_MUL) {
#pragma unroll
                for (int e = 0; e < 8; e += 2) {
                    const float2 p = __half22float2(__hmul2(silu_h2(__halves2half2(h[e], h[e + 1])), __halves2half2(h2[e], h2[e + 1])));
                    f[e] = p.x;
                    f[e + 1] = p.y;
                }
            } else if (P.mode == I8_GELU_MUL) {
#pragma unroll
                for (int e = 0; e < 8; ++e) f[e] = __half2float(__hmul(gelu_h(h[e]), h2[e]));
            } else {
#pragma unroll
                for (int e = 0; e < 8; ++e) f[e] = __half2float(h[e]);
            }
        }
        float amax = 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) amax = fmaxf(amax, fabsf(f[e]));
#pragma unroll
        for (int s = 1; s < 16; s <<= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, s));      // 16 lanes = one 128-k block
        // power-of-two block scale 2^e with max * 2^e in [2^14, 2^15): fp16 row values within a factor 16 of the block maximum
        // are represented EXACTLY and all scale products are exact -- a unit-vector row returns reconstruct()'s fp16 weights.
        // (the exponent is taken from max * (1 + 2^-15): a maximum that would round up to 2^15 gets the next scale instead)
        const uint32_t ef = (__float_as_uint(amax * 1.000030518f) >> 23) & 0xffu;
        const float inv = amax > 0.f ? __uint_as_float((268u - ef) << 23) : 0.f;
        // round to nearest even through the fp32 adder: bits(x * inv + 1.5 * 2^23) = 0x4B400000 + q, the low 16 bits are q as int16
        uint32_t qb[8], usum = 0u;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            qb[e] = __float_as_uint(fmaf(f[e], inv, 12582912.f));
            usum += qb[e];
        }
        int sum = (int)(usum - 8u * 0x4B400000u);
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2);                                                       // 4 lanes = one slab
        if (valid) {
            // byte planes of (q0, q4, q1, q5) | (q2, q6, q3, q7): high bytes (signed) and low bytes (unsigned)
            auto pack = [&](int i0, int i1, int i2, int i3, uint32_t sel) -> uint32_t {
                return __byte_perm(__byte_perm(qb[i0], qb[i1], sel), __byte_perm(qb[i2], qb[i3], sel), 0x5410u);
            };
            uint2 hw, lw;
            hw.x = pack(0, 4, 1, 5, 0x0051u); hw.y = pack(2, 6, 3, 7, 0x0051u);
            lw.x = pack(0, 4, 1, 5, 0x0040u); lw.y = pack(2, 6, 3, 7, 0x0040u);
            const int si = o >> 2, j = o & 3;
            *reinterpret_cast<uint2*>(act_g + (size_t)si * 64 + j * 8) = hw;
            *reinterpret_cast<uint2*>(act_g + (size_t)si * 64 + 32 + j * 8) = lw;
            if (j == 0) asum_s[si] = sum;
            if ((o & 15) == 0) ascale_s[si >> 2] = amax > 0.f ? __uint_as_float((ef - 14u) << 23) : 0.f;
        }
    };
#pragma unroll
    for (int r = 0; r < PF; ++r)
        if (r * I8_THREADS < n_oct) stage_round(r * I8_THREADS + tid, pv[r], wv[r], smem_gather, hg[r]);
    for (int ob = PF * I8_THREADS; ob < n_oct; ob += I8_THREADS) {
        const int o = ob + tid;
        uint4 pidx = make_uint4(0, 0, 0, 0), wreg = make_uint4(0, 0, 0, 0);
        if (o < n_oct) {
            if (P.perm && (gather_x || !P.norm_permuted)) pidx = __ldg(reinterpret_cast<const uint4*>(P.perm + o * 8));
            if (P.mode == I8_RMSNORM) {
                if (P.perm && !P.norm_permuted) {
                    const uint16_t* pi = reinterpret_cast<const uint16_t*>(&pidx);
                    uint16_t* wo = reinterpret_cast<uint16_t*>(&wreg);
#pragma unroll
                    for (int e = 0; e < 8; ++e) wo[e] = __half_as_ushort(__ldg(P.norm_w + pi[e]));
                } else {
                    wreg = __ldg(reinterpret_cast<const uint4*>(P.norm_w + o * 8));
                }
            }
        }
        stage_round(o, pidx, wreg, false, make_uint4(0, 0, 0, 0));
    }
    if (P.mode == I8_RMSNORM) {
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) sumsq += __shfl_xor_sync(0xffffffffu, sumsq, s);
        if (lane == 0) s_red[warp] = sumsq;
    }
    __syncthreads();
    EXL2B_STAMP(P, 3);
    float rrms = 1.f;
    if (P.mode == I8_RMSNORM) {
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < I8_WARPS; ++i) t += s_red[i];
        rrms = rsqrtf(t * (1.0f / (float)P.K) + P.norm_eps);
    }

    // what this warp needs to finish block (warp) of the CTA after the main loop -- who holds its partial sums, where the result goes,
    // bias / old value for the residual add -- is fetched now, so that the tail of the launch waits for no load
    uint32_t red0 = 0u;
    I8OutPre opre0 = {0u, 0u};
    if (warp < nb) {
        red0 = __ldg(P.plan_red + blk0 + warp);
        if (red0 & 0xffffu) opre0 = out_pre(P, blk0 + warp, lane);
    }

    // ---- main loop: this warp alone, stage by stage; everything positional comes from the stage list.
    int am[4] = {0, 0, 0, 0}, ae[2] = {0, 0};
    float tot = 0.f;
    int S = 0, blk_slabs = 0, emits = 0;
#pragma unroll 1
    for (int s = 0; s < nst; ++s) {
        const uint4 d = lds128(lwin + ((uint32_t)s & (I8_LWIN - 1)) * 16u);
        const int nreq = (int)((d.w >> 24) & 15u);
        const uint32_t slot8 = (uint32_t)s & (I8_BARS - 1);
        mbar_wait(bar0 + slot8 * 8u, ((uint32_t)s >> 3) & 1u);
        const int ks = (int)(d.z & 0x7ffu), n = (int)((d.z >> 11) & 7u), bits = (int)((d.z >> 14) & 15u);
        const uint32_t slot = ring + ((d.w >> 16) & 0xffu) * 128u;
        const uint32_t xs = act + (uint32_t)ks * 64u, as = asum + (uint32_t)ks * 4u;
        {   // dispatch on the bit width as a chain of warp-uniform branches, most frequent first.  (`opaque` keeps the compiler from
            // fusing the chain into a jump table: BRX through a constant-bank table costs a dependent LDC per stage)
            int bsel = bits;
            auto opaque = [&]() { asm volatile("" : "+r"(bsel)); return bsel; };
            if (bsel == 4) S += consume_stage<4>(slot, n, xs, as, lane, am, ae);
            else if (opaque() == 5) S += consume_stage<5>(slot, n, xs, as, lane, am, ae);
            else if (opaque() == 6) S += consume_stage<6>(slot, n, xs, as, lane, am, ae);
            else if (opaque() == 3) S += consume_stage<3>(slot, n, xs, as, lane, am, ae);
            else if (opaque() == 8) S += consume_stage<8>(slot, n, xs, as, lane, am, ae);
            else S += consume_stage<2>(slot, n, xs, as, lane, am, ae);
        }
        // what this stage's barrier delivered besides the weights: the descriptors of the stages its space will be given to,
        // and (flush stages) this lane's scale -- read before the requests below may overwrite the scale slot
        uint4 dreq = make_uint4(0u, 0u, 0u, 0u);
        if (lane < nreq) dreq = lds128(lwin + ((uint32_t)(next_req + lane) & (I8_LWIN - 1)) * 16u);
        uint32_t wraw = 0u;
        if (d.z & (DF_FLUSH << 18))
            wraw = (d.z & (DF_GPTQ << 18)) ? lds32(sring + slot8 * (uint32_t)P.srow + (uint32_t)lane * 4u)
                                           : lds_u16(sring + slot8 * (uint32_t)P.srow + (uint32_t)lane * 2u);
        __syncwarp();
        {                                          // the space this stage occupied is free: request the stages waiting for it
            issue_stages(next_req, nreq, dreq);
            next_req += nreq;
        }
        blk_slabs += n;
        if (d.z & (DF_FLUSH << 18)) {
            // integer sums -> fp32:  sum_k a_k (q_k - zero) * scale  =  (sum a q - zero * sum a) * scale_w * scale_row
            int v = ((am[0] << 8) + am[1]) + (((am[2] << 8) + am[3]) >> 4) + (((ae[0] << 8) + ae[1]) << plane_main(bits));
            const float ws = __half2float(__ushort_as_half((unsigned short)(wraw & 0xffffu)));
            const int zero = (d.z & (DF_GPTQ << 18)) ? (int)(wraw >> 16) : (1 << (bits - 1));
            v -= zero * S;
            tot = fmaf((float)v, ws * __uint_as_float(lds32(ascale + (uint32_t)(ks >> 2) * 4u)), tot);
            am[0] = am[1] = am[2] = am[3] = 0;
            ae[0] = ae[1] = 0;
            S = 0;
            if (d.z & (DF_BLOCK_DONE << 18)) {
                const int blk = blk0 + (int)(d.w & 0xffffu);
                if (blk_slabs == KS) {
                    finalize_block(P, blk, lane, out_pre(P, blk, lane), tot * rrms);          // this warp covered the block's whole K by itself
                } else {
                    if (emits >= 2) __trap();       // a warp's range has at most two partial blocks (its first and its last)
                    emit_base[(warp * 2 + emits) * 32 + lane] = tot;
                    ++emits;
                }
                tot = 0.f;
                blk_slabs = 0;
            }
        }
    }
    EXL2B_STAMP(P, 4);
    __syncthreads();
    EXL2B_STAMP(P, 5);

    // ---- split-K never left the CTA: sum the warps' partials of each block in warp order (the plan says which warps hold them),
    //      finalise.  Blocks covered by one warp alone were finalised in the main loop (no partials).
    for (int b = warp; b < nb; b += I8_WARPS) {
        const uint32_t rd = (b == warp) ? red0 : __ldg(P.plan_red + blk0 + b);
        uint32_t m = rd & 0xffffu;
        if (m == 0u) continue;
        int w = __ffs(m) - 1;
        float v = emit_base[(w * 2 + (int)((rd >> 16) & 1u)) * 32 + lane];
        for (m &= m - 1u; m; m &= m - 1u) {
            w = __ffs(m) - 1;
            v += emit_base[(w * 2) * 32 + lane];
        }
        finalize_block(P, blk0 + b, lane, (b == warp) ? opre0 : out_pre(P, blk0 + b, lane), v * rrms);
    }
    if (tid == 0) slot_release(P.slot_cnt);
    if (P.dbg && lane == 0) atomicMax(P.dbg + 7, globaltimer());
    if (P.dbg_rec && tid == 0 && blockIdx.x < 160) {
        unsigned smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        P.dbg_rec[blockIdx.x * 4 + 2] = globaltimer();
        P.dbg_rec[blockIdx.x * 4 + 3] = smid;
    }
}

// ---- host side ---------------------------------------------------------------------------------------------------------------

bool gemv_i8_enabled() {
    static const bool on = [] {
        const char* e = getenv("EXL2B_GEMV");
        return !(e && e[0] == 't');
    }();
    return on;
}

bool gemv_i8_fusable(const QMatrix* const* qs, int nm) {
    if (nm < 1 || nm > I8_MAX_MATS) return false;
    for (int i = 0; i < nm; ++i) {
        if (!qs[i] || qs[i]->v.layout != LAYOUT_TC || qs[i]->v.K != qs[0]->v.K || qs[i]->device != qs[0]->device) return false;
        if ((qs[i]->v.perm == nullptr) != (qs[0]->v.perm == nullptr)) return false;
    }
    if (nm == 1 || !qs[0]->v.perm) return true;
    const int K = qs[0]->v.K;
    std::vector<uint16_t> p0(K), pi(K);
    if (cudaSetDevice(qs[0]->device) != cudaSuccess) return false;
    if (cudaMemcpy(p0.data(), qs[0]->v.perm, (size_t)K * 2, cudaMemcpyDeviceToHost) != cudaSuccess) return false;
    for (int i = 1; i < nm; ++i) {
        if (qs[i]->v.perm == qs[0]->v.perm) continue;
        if (cudaMemcpy(pi.data(), qs[i]->v.perm, (size_t)K * 2, cudaMemcpyDeviceToHost) != cudaSuccess) return false;
        if (p0 != pi) return false;
    }
    return true;
}

// Contiguous partition of the launch's blocks over at most `ctas` CTAs minimising the largest CTA (in bytes).
void i8_partition_blocks(const std::vector<uint32_t>& bytes, int ctas, unsigned short* out, int* used) {
    const int nb = (int)bytes.size();
    unsigned long long total = 0, biggest = 0;
    for (uint32_t b : bytes) { total += b; biggest = std::max<unsigned long long>(biggest, b); }
    unsigned long long lo = std::max(biggest, (total + ctas - 1) / ctas), hi = total;
    auto fits = [&](unsigned long long cap) {
        int c = 1;
        unsigned long long acc = 0;
        for (uint32_t b : bytes) {
            if (acc + b > cap) { ++c; acc = 0; }
            acc += b;
        }
        return c <= ctas;
    };
    while (lo < hi) {
        const unsigned long long mid = (lo + hi) / 2;
        if (fits(mid)) hi = mid; else lo = mid + 1;
    }
    int c = 0;
    unsigned long long acc = 0;
    out[0] = 0;
    for (int b = 0; b < nb; ++b) {
        if (acc + bytes[b] > lo) { out[++c] = (unsigned short)b; acc = 0; }
        acc += bytes[b];
    }
    out[++c] = (unsigned short)nb;
    *used = c;
}

// RMSNorm weight in a matrix' stored-row order.  Only a block handle keeps such a copy, made when the handle is created (as
// the reference's handles take their tensors at creation); a bare call gathers the weight in the kernel, so no copy can
// outlive or lag behind the weight it was made from.
__global__ void gather_rows_kernel(half* __restrict__ out, const half* __restrict__ w, const uint16_t* __restrict__ perm, int K) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < K) out[i] = w[perm[i]];
}
int permuted_norm_copy(const QMatrix* q, const half* norm_w, half** out) {
    *out = nullptr;
    half* p = nullptr;
    EXL2B_CUDA(cudaDeviceSynchronize());             // the weight may still be in flight on any stream
    EXL2B_CUDA(cudaMalloc(&p, (size_t)q->v.K * sizeof(half)));
    gather_rows_kernel<<<(q->v.K + 255) / 256, 256>>>(p, norm_w, q->v.perm, q->v.K);
    g_launch_count++;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        cudaFree(p);
        EXL2B_CUDA(e);
    }
    *out = p;
    return 0;
}

// ---- launch plans -------------------------------------------------------------------------------------------------------
// Everything positional about a launch (block -> CTA partition, every warp's stage list) depends only on the STRUCTURE of its
// matrices (K, N, bit-width regions, group sizes), not on their addresses: it is computed here once per structure, uploaded,
// and shared by every launch with that structure (all 32 layers of a model use the same few plans, so the descriptors stay in
// L2).  The kernel reads its list with one coalesced load per warp: no region walk, no divisions, no dynamic indexing of kernel
// parameters on the device.
struct I8Plan {
    uint4* d_desc = nullptr;
    uint32_t* d_first = nullptr;
    uint32_t* d_cta = nullptr;
    uint32_t* d_red = nullptr;
    int ctas = 0, lcap = 0, arena = 0, srow = 64;
};
struct I8PlanMat {
    int N, KS, is_gptq, num_regions;
    uint32_t blk_stream_bytes;
    QRegion reg[MAX_REGIONS];
};
static std::map<std::string, I8Plan> g_plans[64];
static std::mutex g_plan_mutex;

// stage lists of one launch structure: the same walk for every (CTA, warp) -- units are (block, slab) pairs, CTA-relative
static void i8_build_lists(const I8PlanMat* mats, int nm, const unsigned short* cta_blk, int C, int warps, int arena,
                           std::vector<uint4>& desc, std::vector<uint32_t>& first, std::vector<uint32_t>& cta, std::vector<uint32_t>& red,
                           int* lcap) {
    const int KS = mats[0].KS;
    int blk_base[I8_MAX_MATS + 1] = {0};
    for (int i = 0; i < nm; ++i) blk_base[i + 1] = blk_base[i] + (mats[i].N + 31) / 32;
    *lcap = 1;
    red.assign(blk_base[nm], 0u);
    for (int c = 0; c < C; ++c) {
        const int blk0 = cta_blk[c], nb = (int)cta_blk[c + 1] - blk0;
        cta.push_back((uint32_t)blk0 | ((uint32_t)nb << 16));
        const long long units = (long long)nb * KS;
        for (int w = 0; w < warps; ++w) {
            first.push_back((uint32_t)desc.size());
            const int l0 = (int)((units * w) / warps), l1 = (int)((units * (w + 1)) / warps);
            int lin = l0;
            while (lin < l1) {
                const int b = lin / KS, ks = lin - b * KS, blk = blk0 + b;
                int mi = 0;
                while (mi + 1 < nm && blk >= blk_base[mi + 1]) ++mi;
                const I8PlanMat& m = mats[mi];
                int r = 0;
                while (r + 1 < m.num_regions && ks >= m.reg[r + 1].ks_begin) ++r;
                const QRegion& rg = m.reg[r];
                const int r_end = (r + 1 < m.num_regions) ? m.reg[r + 1].ks_begin : KS;
                const int rel = ks - rg.ks_begin, g = rel >> rg.spg_log2;
                const int gend = rg.ks_begin + ((g + 1) << rg.spg_log2);
                // a stage never crosses a quantisation group, a 128-k row block, a bit-width region or the end of the warp's range
                const int segend = std::min(std::min(gend, (ks | 3) + 1), std::min(r_end, ks + (l1 - lin)));
                const int len = segend - ks, cap = std::max(1, std::min(4, (arena / 2) / (128 * rg.bits)));
                const int pieces = (len + cap - 1) / cap, n = (len + pieces - 1) / pieces;
                uint32_t flags = (ks + n == segend ? DF_FLUSH : 0u) | ((ks + n == KS || lin + n == l1) ? DF_BLOCK_DONE : 0u) | (m.is_gptq ? DF_GPTQ : 0u);
                if (flags & DF_BLOCK_DONE) flags |= DF_FLUSH;
                const int bim = blk - blk_base[mi];
                uint4 d;
                d.x = (uint32_t)bim * m.blk_stream_bytes + rg.off_base + (uint32_t)rel * 128u * (uint32_t)rg.bits;
                d.y = (uint32_t)(rg.group_base + g) * (uint32_t)m.N + (uint32_t)bim * 32u;
                d.z = (uint32_t)ks | ((uint32_t)n << 11) | ((uint32_t)rg.bits << 14) | (flags << 18) | ((uint32_t)mi << 22) |
                      ((uint32_t)(n * rg.bits) << 24);          // (bytes / 128 <= 32)
                d.w = (uint32_t)b;
                desc.push_back(d);
                lin += n;
            }
            // partial sums this warp leaves in shared memory (the kernel's `emits` counter, replayed): per block the set of such warps
            // and which of its two partial slots the first one uses (every later warp starts inside the block: slot 0)
            {
                int slabs = 0, emits = 0;
                for (size_t s = first.back(); s < desc.size(); ++s) {
                    const uint4& d = desc[s];
                    slabs += (int)((d.z >> 11) & 7u);
                    if (((d.z >> 18) & 15u) & DF_BLOCK_DONE) {
                        if (slabs != KS) {
                            uint32_t& r = red[blk0 + (int)(d.w & 0xffffu)];
                            if ((r & 0xffffu) == 0) r = (uint32_t)emits << 16;          // the first warp may be on its second partial
                            r |= 1u << w;
                            ++emits;
                        }
                        slabs = 0;
                    }
                }
            }
            // place the warp's stages in its byte arena (a ring): `req` of stage c = how many later stages may be requested once c
            // has been consumed; n_pre = how many are requested up front.  At most I8_BARS stages are ever in flight.
            const size_t w0 = first.back(), nst = desc.size() - w0;
            *lcap = std::max(*lcap, (int)nst);
            std::vector<int> dep(nst, -1);
            {
                struct Live { int idx; uint32_t off, size; };
                std::vector<Live> live;
                uint32_t off = 0;
                int last_dep = -1;
                for (size_t s = 0; s < nst; ++s) {
                    const uint4& d = desc[w0 + s];
                    const uint32_t size = ((d.z >> 11) & 7u) * ((d.z >> 14) & 15u) * 128u;
                    if (off + size > (uint32_t)arena) off = 0;
                    auto overlaps = [&](const Live& l) { return l.off < off + size && off < l.off + l.size; };
                    for (;;) {
                        bool hit = false;
                        for (const Live& l : live) hit = hit || overlaps(l);
                        if (!hit && (int)live.size() < I8_BARS) break;
                        last_dep = live.front().idx;          // consumption is in order: free the oldest
                        live.erase(live.begin());
                    }
                    dep[s] = last_dep;
                    live.push_back(Live{(int)s, off, size});
                    desc[w0 + s].w |= (off / 128u) << 16;
                    off += size;
                }
            }
            int n_pre = 0;
            for (size_t s = 0; s < nst; ++s) {
                if (dep[s] < 0) ++n_pre;
                else desc[w0 + dep[s]].w += 1u << 24;
            }
            first.back() |= (uint32_t)n_pre << 26;
        }
    }
    first.push_back((uint32_t)desc.size());
}

// the host half of a plan: partition, arena size, scale-slot size and stage lists of one launch structure on `sms` CTAs
static int i8_plan_host(const I8PlanMat* mats, int nm, int sms, int warps, I8Plan& pl, std::vector<uint4>& desc,
                        std::vector<uint32_t>& first, std::vector<uint32_t>& cta, std::vector<uint32_t>& red) {
    std::vector<uint32_t> blk_bytes;
    for (int i = 0; i < nm; ++i) {
        // only blocks that hold real columns (the last strip of a padded matrix may contain all-padding blocks)
        for (int b = 0; b < (mats[i].N + 31) / 32; ++b) blk_bytes.push_back(mats[i].blk_stream_bytes);
    }
    EXL2B_REQUIRE(blk_bytes.size() < 65535, "too many column blocks (%zu)", blk_bytes.size());
    EXL2B_REQUIRE((long long)blk_bytes.size() * mats[0].KS < (1ll << 30), "problem too large for 32-bit unit arithmetic");
    unsigned short cta_blk[I8_MAX_CTAS + 1];
    i8_partition_blocks(blk_bytes, sms, cta_blk, &pl.ctas);
    // two launches co-resident per SM (227 KB, 1 KB reserved per CTA) is what lets the next launch prefetch: a CTA gets at most
    // 111 KB of dynamic shared memory (EXL2B_I8_SMEM overrides), and what the staged row / lists leave of it is split into the warps' weight arenas
    static const int smem_budget = [] { const char* e = getenv("EXL2B_I8_SMEM"); return e ? atoi(e) : 111 * 1024; }();
    pl.srow = 64;
    for (int i = 0; i < nm; ++i)
        if (mats[i].is_gptq) pl.srow = 128;
    pl.arena = 8192;
    for (;;) {
        desc.clear(); first.clear(); cta.clear();
        i8_build_lists(mats, nm, cta_blk, pl.ctas, warps, pl.arena, desc, first, cta, red, &pl.lcap);
        if ((int)i8_smem_map(warps, pl.arena, mats[0].KS, pl.srow).total <= smem_budget || pl.arena <= 2048) break;
        pl.arena -= 128;
    }
    EXL2B_REQUIRE(desc.size() < (1u << 26), "too many stages");
    return 0;
}

static int i8_get_plan(int device, const I8PlanMat* mats, int nm, int sms, int warps, I8Plan* out) {
    std::string key((const char*)mats, sizeof(I8PlanMat) * nm);
    const int extra[3] = {nm, sms, warps};
    key.append((const char*)extra, sizeof(extra));
    std::lock_guard<std::mutex> lk(g_plan_mutex);
    auto it = g_plans[device].find(key);
    if (it != g_plans[device].end()) { *out = it->second; return 0; }

    I8Plan pl;
    std::vector<uint4> desc;
    std::vector<uint32_t> first, cta, red;
    const int rc = i8_plan_host(mats, nm, sms, warps, pl, desc, first, cta, red);
    if (rc) return rc;
    EXL2B_CUDA(cudaMalloc(&pl.d_desc, desc.size() * sizeof(uint4) + 16));
    EXL2B_CUDA(cudaMalloc(&pl.d_first, first.size() * 4));
    EXL2B_CUDA(cudaMalloc(&pl.d_cta, cta.size() * 4));
    EXL2B_CUDA(cudaMemcpy(pl.d_desc, desc.data(), desc.size() * sizeof(uint4), cudaMemcpyHostToDevice));
    EXL2B_CUDA(cudaMemcpy(pl.d_first, first.data(), first.size() * 4, cudaMemcpyHostToDevice));
    EXL2B_CUDA(cudaMemcpy(pl.d_cta, cta.data(), cta.size() * 4, cudaMemcpyHostToDevice));
    EXL2B_CUDA(cudaMalloc(&pl.d_red, red.size() * 4 + 4));
    EXL2B_CUDA(cudaMemcpy(pl.d_red, red.data(), red.size() * 4, cudaMemcpyHostToDevice));
    g_plans[device][key] = pl;
    *out = pl;
    return 0;
}

// A launch structure is planned (cudaMalloc + synchronous upload) the first time it is seen: never inside a stream capture --
// run every shape once eagerly first, as model.capture() does.
int gemv_i8_launch(int device, cudaStream_t stream, const I8Out* outs, int nm, const I8Input& in) {
    EXL2B_REQUIRE(nm >= 1 && nm <= I8_MAX_MATS, "bad matrix count %d", nm);
    EXL2B_REQUIRE(device >= 0 && device < 64, "bad device %d", device);
    EXL2B_REQUIRE(in.x, "null input row");
    EXL2B_REQUIRE(in.mode != I8_RMSNORM || in.norm_w, "RMSNorm prologue without a weight");
    EXL2B_REQUIRE((in.mode != I8_SILU_MUL && in.mode != I8_GELU_MUL) || in.x2, "act*mul prologue without the second operand");
    // warps per CTA: 16 (64 registers / thread) or 12 (80) -- EXL2B_I8_WARPS selects, both keep two CTAs per SM resident
    static const int warps = [] {
        const char* e = getenv("EXL2B_I8_WARPS");
        const int w = e ? atoi(e) : 16;
        return (w == 12 || w == 8) ? w : 16;
    }();
    static bool attr_set[64] = {false};
    if (!attr_set[device]) {
        EXL2B_CUDA(cudaFuncSetAttribute(gemv_i8_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        EXL2B_CUDA(cudaFuncSetAttribute(gemv_i8_kernel<12>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        EXL2B_CUDA(cudaFuncSetAttribute(gemv_i8_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr_set[device] = true;
    }

    I8Params P = {};
    P.num_mats = nm;
    P.K = outs[0].q->v.K;
    P.KS = outs[0].q->v.KS;
    P.perm = outs[0].q->v.perm;
    P.x = in.x;
    P.x2 = in.x2;
    P.norm_w = in.norm_w;
    P.norm_eps = in.norm_eps;
    P.mode = in.mode;
    P.x_permuted = in.x_permuted;
    if (in.mode == I8_RMSNORM && P.perm && in.norm_wp) {
        P.norm_w = in.norm_wp;
        P.norm_permuted = 1;
    }
    I8PlanMat pm[I8_MAX_MATS];
    memset(pm, 0, sizeof(pm));
    int blk = 0;
    for (int i = 0; i < nm; ++i) {
        const QMatrix* q = outs[i].q;
        EXL2B_REQUIRE(q && outs[i].c, "null matrix / output");
        const QMatView& v = q->v;
        EXL2B_REQUIRE(v.layout == LAYOUT_TC, "matrix is not in the default (LAYOUT_TC) layout");
        EXL2B_REQUIRE(v.KS == P.KS, "fused matrices must share K");
        EXL2B_REQUIRE((v.perm == nullptr) == (P.perm == nullptr), "fused matrices must share their row permutation");
        EXL2B_REQUIRE(q->wtab, "matrix has no scale table");
        // scale rows are bulk-copied from (group * N + 32 * block) * (2 or 4) bytes: 16-byte aligned because N % 8 == 0, which
        // exl2b_qmatrix_create requires (the reference's q_scale / qzeros pack 8 columns per word)
        EXL2B_REQUIRE(v.N % 8 == 0, "width %d is not a multiple of 8", v.N);
        EXL2B_REQUIRE(q->packed_bytes < (1ull << 32), "matrix too large for 32-bit stage offsets");
        I8Mat& m = P.mat[i];
        m.packed = reinterpret_cast<const uint8_t*>(v.packed);
        m.wtab = q->wtab;
        m.bias = v.bias;
        m.c = outs[i].c;
        m.c_perm = outs[i].c_perm;
        m.out_invperm = outs[i].out_invperm;
        m.clear = outs[i].clear;
        m.N = v.N;
        m.blk_base = blk;
        blk += (v.N + 31) / 32;
        pm[i].N = v.N;
        pm[i].KS = v.KS;
        pm[i].is_gptq = v.is_gptq;
        pm[i].num_regions = v.num_regions;
        pm[i].blk_stream_bytes = v.blk_stream_bytes;
        for (int r = 0; r < v.num_regions; ++r) pm[i].reg[r] = v.reg[r];
    }
    EXL2B_REQUIRE(P.KS <= 2048, "K = %d exceeds the stage descriptor (K <= 65536)", P.K);
    I8Plan pl;
    // EXPERIMENT (EXL2B_I8_DOUBLE_MB=n, off by default): launches of at least n MB use BOTH slots of every SM themselves (twice the
    // CTAs, half the work each: 32 warps per SM on one launch) instead of leaving one to the next launch's prefetch
    static const int double_mb = [] { const char* e = getenv("EXL2B_I8_DOUBLE_MB"); return e ? atoi(e) : 0; }();
    unsigned long long launch_bytes = 0;
    for (int i = 0; i < nm; ++i) launch_bytes += outs[i].q->packed_bytes;
    const int slots = (double_mb > 0 && launch_bytes >= (unsigned long long)double_mb << 20) ? 2 : 1;
    const int grid_ctas = std::min(device_sm_count(device) * slots, I8_MAX_CTAS);
    int rc = i8_get_plan(device, pm, nm, grid_ctas, warps, &pl);
    if (rc) return rc;
    P.plan_desc = pl.d_desc;
    P.plan_first = pl.d_first;
    P.plan_cta = pl.d_cta;
    P.plan_red = pl.d_red;
    P.arena = pl.arena;
    P.srow = pl.srow;
    P.busy_ctas = pl.ctas;
    static const int l2pf = [] { const char* e = getenv("EXL2B_I8_L2PF"); return e ? atoi(e) : 0; }();
    P.l2_prefetch = l2pf;
    const size_t smem_total = i8_smem_map(warps, P.arena, P.KS, P.srow).total;
    EXL2B_REQUIRE(smem_total <= 200 * 1024, "shared memory budget exceeded (%zu bytes, K = %d)", smem_total, P.K);
    extern unsigned long long* g_dbg;
    extern int g_dbg_cta, g_dbg_slot;
    P.dbg = g_dbg ? g_dbg + 32 * (g_dbg_slot++ % 64) : nullptr;
    P.dbg_cta = g_dbg_cta;
    extern unsigned long long* g_dbg_rec;
    P.dbg_rec = (g_dbg_rec && P.dbg) ? g_dbg_rec + (size_t)((g_dbg_slot - 1) % 64) * 160 * 4 : nullptr;      // [64][160][4], CTAs 0..159
    // one CTA per SM, always (slot holders, see the kernel); a self-resetting counter per launch in flight
    static SlotCounters slot_cnts;
    rc = next_slot_counter(slot_cnts, device, &P.slot_cnt);
    if (rc) return rc;
    const int C = slot_holders_disabled() ? pl.ctas : std::max(pl.ctas, grid_ctas);
    if (warps == 16) EXL2B_CUDA(launch_pdl_f("i8", gemv_i8_kernel<16>, dim3(C), dim3(16 * 32), smem_total, stream, P));
    else if (warps == 12) EXL2B_CUDA(launch_pdl_f("i8", gemv_i8_kernel<12>, dim3(C), dim3(12 * 32), smem_total, stream, P));
    else EXL2B_CUDA(launch_pdl_f("i8", gemv_i8_kernel<8>, dim3(C), dim3(8 * 32), smem_total, stream, P));
    return 0;
}

}  // namespace exl2b

extern "C" int exl2b_row_gemv_i8(void) { return exl2b::gemv_i8_enabled() ? 1 : 0; }

// host-only diagnostics hook (tests/test_i8_emulation.py): the block -> CTA partition gemv_i8_launch would use
extern "C" int exl2b_debug_partition(const uint32_t* block_bytes, int num_blocks, int ctas, uint16_t* out, int* used) {
    EXL2B_REQUIRE(block_bytes && out && used && num_blocks > 0 && ctas > 0 && ctas <= exl2b::I8_MAX_CTAS, "bad argument");
    std::vector<uint32_t> b(block_bytes, block_bytes + num_blocks);
    exl2b::i8_partition_blocks(b, ctas, out, used);
    return 0;
}

// host-only diagnostics hook (tests/test_i8_emulation.py): the stage lists gemv_i8_launch would use for ONE matrix with the
// given regions (5 ints each: ks_begin, bits, spg_log2, group_base, off_base).  desc: capacity cap_desc x 4 words; first:
// ctas * warps + 1 words; returns the CTA count in *ctas_used, the descriptor count in *n_desc.
extern "C" int exl2b_debug_plan(int N, int KS, int is_gptq, uint32_t blk_stream_bytes, const int* regions, int num_regions, int ctas, int warps,
                                int slot_bytes, uint32_t* desc, int cap_desc, uint32_t* first, int* ctas_used, int* n_desc, int* lcap,
                                uint32_t* red) {
    EXL2B_REQUIRE(regions && desc && first && ctas_used && n_desc && lcap, "null argument");
    EXL2B_REQUIRE(num_regions >= 1 && num_regions <= exl2b::MAX_REGIONS && ctas > 0 && ctas <= exl2b::I8_MAX_CTAS && warps > 0, "bad argument");
    exl2b::I8PlanMat m;
    memset(&m, 0, sizeof(m));
    m.N = N; m.KS = KS; m.is_gptq = is_gptq; m.num_regions = num_regions; m.blk_stream_bytes = blk_stream_bytes;
    for (int r = 0; r < num_regions; ++r)
        m.reg[r] = exl2b::QRegion{regions[5 * r], regions[5 * r + 1], regions[5 * r + 2], regions[5 * r + 3], (uint32_t)regions[5 * r + 4]};
    std::vector<uint32_t> bb((N + 31) / 32, blk_stream_bytes);
    unsigned short cta_blk[exl2b::I8_MAX_CTAS + 1];
    exl2b::i8_partition_blocks(bb, ctas, cta_blk, ctas_used);
    std::vector<uint4> d;
    std::vector<uint32_t> f, c, r;
    exl2b::i8_build_lists(&m, 1, cta_blk, *ctas_used, warps, slot_bytes, d, f, c, r, lcap);      // slot_bytes = bytes of a warp's arena
    EXL2B_REQUIRE((int)d.size() <= cap_desc, "descriptor buffer too small (%zu)", d.size());
    memcpy(desc, d.data(), d.size() * sizeof(uint4));
    memcpy(first, f.data(), f.size() * 4);
    if (red) memcpy(red, r.data(), r.size() * 4);          // [ceil(N / 32)]
    *n_desc = (int)d.size();
    return 0;
}

// host-only diagnostics hook (tests/test_i8_smem_operands.py): the whole plan gemv_i8_launch would make for a launch of nm fused
// matrices on `ctas` CTAs of `warps` warps.  mats: per matrix 5 + 5 * MAX_REGIONS ints (N, KS, is_gptq, blk_stream_bytes,
// num_regions, then per region ks_begin, bits, spg_log2, group_base, off_base).  desc: capacity cap_desc x 4 words; first:
// capacity cap_first words.  info: [0] CTAs with blocks, [1] descriptors, [2] arena bytes per warp, [3] scale-slot bytes,
// [4] dynamic shared memory of a CTA, [5] longest stage list.
extern "C" int exl2b_debug_i8_plan(const int* mats, int nm, int ctas, int warps, uint32_t* desc, int cap_desc, uint32_t* first,
                                   int cap_first, int* info) {
    EXL2B_REQUIRE(mats && desc && first && info, "null argument");
    EXL2B_REQUIRE(nm >= 1 && nm <= exl2b::I8_MAX_MATS && ctas > 0 && ctas <= exl2b::I8_MAX_CTAS && warps > 0, "bad argument");
    exl2b::I8PlanMat pm[exl2b::I8_MAX_MATS];
    memset(pm, 0, sizeof(pm));
    for (int i = 0; i < nm; ++i) {
        const int* r = mats + i * (5 + 5 * exl2b::MAX_REGIONS);
        EXL2B_REQUIRE(r[4] >= 1 && r[4] <= exl2b::MAX_REGIONS && r[1] == mats[1], "bad matrix %d", i);
        pm[i].N = r[0]; pm[i].KS = r[1]; pm[i].is_gptq = r[2]; pm[i].blk_stream_bytes = (uint32_t)r[3]; pm[i].num_regions = r[4];
        for (int g = 0; g < r[4]; ++g) {
            const int* q = r + 5 + 5 * g;
            pm[i].reg[g] = exl2b::QRegion{q[0], q[1], q[2], q[3], (uint32_t)q[4]};
        }
    }
    exl2b::I8Plan pl;
    std::vector<uint4> d;
    std::vector<uint32_t> f, c, red;
    const int rc = exl2b::i8_plan_host(pm, nm, ctas, warps, pl, d, f, c, red);
    if (rc) return rc;
    EXL2B_REQUIRE((int)d.size() <= cap_desc && (int)f.size() <= cap_first, "output buffers too small (%zu, %zu)", d.size(), f.size());
    memcpy(desc, d.data(), d.size() * sizeof(uint4));
    memcpy(first, f.data(), f.size() * 4);
    info[0] = pl.ctas;
    info[1] = (int)d.size();
    info[2] = pl.arena;
    info[3] = pl.srow;
    info[4] = (int)exl2b::i8_smem_map(warps, pl.arena, pm[0].KS, pl.srow).total;
    info[5] = pl.lcap;
    return 0;
}
