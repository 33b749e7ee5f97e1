// wgmma dequant-GEMM: packed EXL2 / GPTQ weights -> fp16 tiles in shared memory -> wgmma against the activations.
// Serves 2..16 rows (and single rows when the integer GEMV is switched off) in 8-row passes, and chained launches of up to 64
// rows in one pass (LAYOUT_TC matrices); replaces gemm_half_q_half_kernel (exllamav2_ext/cuda/q_gemm_kernel.cuh:140-565) and
// gemm_half_q_half_gptq_kernel (q_gemm_kernel_gptq.cuh:61-246).  Un-chained launches above GEMM_BIG_MIN_ROWS = 16 rows take the
// reconstruct + dense GEMM path instead (gemm_big.cu).
//
// The weights are the M operand and the tokens the N operand of the warpgroup MMA:
//     D[128 weight columns x TW tokens] += A[128 x 16 k] (shared memory) * B[16 k x TW tokens] (shared memory)
// two wgmma.m64nTWk16 per 16 k cover a 128-column strip, so the tensor core does every multiply-add and the CUDA cores only
// unpack (3 SHF + 4 LOP3 per 8 four-bit weights) and store the fp16 tile (one STS.128 per 8 weights of a column).
// The token tile TW is the narrowest of 8, 32 and 64 that holds a launch's rows (tc_tile): 1..8 rows run the 8-wide kernels
// (2 CTAs per SM), 9..32 and 33..64 rows (chained launches only) the 32- and 64-wide ones, whose accumulators (TW / 2 fp32
// per M tile and thread, twice: the group's sums and the running totals) and 8-16 KB activation stages need one CTA per SM.
//
// Mapping (layout.h, LAYOUT_TC): strip = 128 output columns = the 128 rows of the A tile; during the unpack a thread IS a
// weight column n.
//   * 256 threads = 2 warpgroups (WG).  Warp w of a WG streams ITS 32-column block of the strip with cp.async.bulk (TMA 1-D)
//     into a private ring, exactly one quantisation group (<= 128 k) per stage.  WG0 takes the first half of a CTA's groups,
//     WG1 the second: two independent software pipelines sharing the tensor core.
//   * per slab (32 k): unpack into 16 half2 registers, store them as row n of the WG's A tile (no-swizzle K-major core
//     matrices, two tiles in turn), fence.proxy.async + WG barrier, four wgmma (2 M tiles x 2 k steps) + commit.  The MMAs
//     of one slab run while the next slab is unpacked; wgmma.wait_group 1 guards the tile before it is written again.
//   * per group: wgmma.wait_group 0, then every thread applies the group's fp16 scales in fp32 to its accumulator fragment
//     (4 columns x TW / 4 tokens) and adds into running totals; the group's stages get the next request.
//   * activations: prepared once per launch by tc_prep_kernel (or scattered there by the producing launch) in the
//     core-matrix layout the B descriptor reads ([k / 8][TW tokens][k % 8]), and fetched per group with one bulk copy per WG.
//   * epilogue: the fragments of both WGs are summed through shared memory into thread = column order; split-K across CTAs
//     and the bias / residual / silu(gate)*up / RoPE epilogues follow row by row (fixed order, deterministic).
#include <algorithm>
#include <mutex>
#include <type_traits>

#include "dequant.cuh"
#include "gemv.cuh"

namespace exl2b {

constexpr int TC_THREADS = 256;                   // 8 unpack warps = 2 warpgroups, each issuing its own wgmma
constexpr int TC_WARPS = 8;
constexpr int TC_MAX_STAGES = 4;                  // stage = one group (<= 4 slabs) of one 32-column block; count + size set per launch
constexpr int TC_NBARS = TC_WARPS * TC_MAX_STAGES + 2 * TC_MAX_STAGES;   // weights | activations
constexpr int TC_SMEM_BARS = TC_NBARS * 8;
constexpr int TC_A_BUFS = 2;                      // per WG: A tiles of one slab, used in turn
constexpr int TC_A_BYTES = 128 * SLAB_K * 2;      // 128 columns x 32 k fp16: 4 planes of 8 k, each 16 core matrices of 8 rows
constexpr int TC_SMEM_CAP = 200 * 1024;           // dynamic shared memory of one CTA, every instantiation
// Sizes that follow the token tile TW (8, 32 or 64; tc_tile):
constexpr int tc_act_stage(int tw) { return 128 * tw * 2; }       // activations of one group: 128 k x TW tokens fp16
constexpr int tc_misc_bytes(int tw) { return tw > GEMV_MTOK ? 128 + 4 * tw : 128; }   // flag; rstd[TW] (at 16, or 128 when wide)
constexpr int tc_ssq_bytes(int tw) { return 4 * tw * 4; }         // [4 warps][TW] per-warp sums of squares
constexpr int tc_corr_floats(int tw) { return 2 * 2 * 4 * 2 * tw; }   // [group parity][WG][warp][S1[TW] | S0[TW]]
constexpr int tc_red_floats(int tw) { return tw * 128; }          // workspace floats per (strip, contributor)
constexpr int tc_comb_bytes(int tw) { return 2 * tw * 128 * 4 + tw * 128 * 2; }   // [2 WG][TW][128] fp32 totals | [TW][128] fp16
// The 8-wide kernels keep the combine buffer in the header; the wide ones overlay it on the pipeline area (activation rings,
// A tiles, weight rings), which is idle once both warpgroups have drained their groups.
constexpr bool tc_comb_overlaid(int tw) { return tw > GEMV_MTOK; }
constexpr int tc_header_bytes(int tw) {
    return (TC_SMEM_BARS + tc_misc_bytes(tw) + (tc_comb_overlaid(tw) ? 0 : tc_comb_bytes(tw)) + tc_ssq_bytes(tw) +
            tc_corr_floats(tw) * 4 + 1023) / 1024 * 1024;
}

// ---- PTX wrappers ----------------------------------------------------------------------------------------------------
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from touching an accumulator between its wgmma and the wait that completes it
template <int N>
__device__ __forceinline__ void wg_fence_acc(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; i += 4) asm volatile("" : "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])::"memory");
}
// D (+)= A[smem desc] * B[smem desc];  M = 64, N = TW, K = 16, fp16 in, fp32 accumulate, both operands K-major.  Fragment d[i]:
// row lane / 4 + 8 ((i >> 1) & 1) of the warp's 16, token 8 (i >> 2) + 2 (lane % 4) + (i & 1)
__device__ __forceinline__ void wgmma_tile(float (&d)[4], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %6, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 {%0, %1, %2, %3}, %4, %5, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}
__device__ __forceinline__ void wgmma_tile(float (&d)[16], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}
__device__ __forceinline__ void wgmma_tile(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}
// one lane of a converged warp (the bulk-copy issuer); returns non-zero in the elected lane
__device__ __forceinline__ uint32_t elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t"
        ".reg .pred px;\n\t"
        "elect.sync _|px, 0xFFFFFFFF;\n\t"
        "@px mov.s32 %0, 1;\n\t"
        "}" : "+r"(pred));
    return pred;
}

// shared-memory matrix descriptor of a no-swizzle K-major operand: core matrix = 8 rows x 16 bytes, contiguous (128 B);
// LBO = byte distance between core matrices adjacent in K, SBO = between core matrices adjacent in M / N
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_byte_addr, uint32_t lbo, uint32_t sbo) {
    return (uint64_t)((smem_byte_addr >> 4) & 0x3FFF) | ((uint64_t)((lbo >> 4) & 0x3FFF) << 16) | ((uint64_t)((sbo >> 4) & 0x3FFF) << 32);
}
// A tile of one slab: plane kb (k 8kb .. 8kb+7) at kb * 2048, row n at n * 16 within it
constexpr uint32_t TC_A_PLANE = 128 * 16;

__device__ __forceinline__ int tc_cta_of_unit(unsigned x, unsigned G, unsigned U) { return (int)(((x + 1u) * G - 1u) / U); }
__device__ __forceinline__ int tc_region_of(const QMatView& w, int ks) {
    int r = 0;
#pragma unroll
    for (int i = 1; i < MAX_REGIONS; ++i)
        if (i < w.num_regions && ks >= w.reg[i].ks_begin) r = i;
    return r;
}
__device__ __forceinline__ int tc_region_end(const QMatView& w, int r) { return (r + 1 < w.num_regions) ? w.reg[r + 1].ks_begin : w.KS; }
// first slab of the group that contains slab ks (ks == KS maps to KS)
__device__ __forceinline__ int tc_group_start(const QMatView& w, int ks) {
    if (ks >= w.KS) return w.KS;
    const QRegion& R = w.reg[tc_region_of(w, ks)];
    return R.ks_begin + (((ks - R.ks_begin) >> R.spg_log2) << R.spg_log2);
}

__device__ __forceinline__ half tc_silu_h(half x) {
    half e = hexp(__hneg(x));
    half r = hrcp(__hadd(__float2half(1.0f), e));
    return __hmul(x, r);
}
__device__ __forceinline__ half tc_gelu_h(half x) {
    float xf = __half2float(x);
    const float c = 0.797884560803f;
    float t = c * (xf + 0.044715f * xf * xf * xf), th;
    asm("tanh.approx.f32 %0, %1;" : "=f"(th) : "f"(t));
    xf = 0.5f * xf * (1.0 + th);
    return __float2half_rn(xf);
}


template <int BITS>
__device__ __forceinline__ void tc_load_words(const uint8_t* base, int lane, uint32_t* mw, uint32_t* ew) {
    constexpr int Pm = plane_main(BITS), Pe = plane_extra(BITS);
    if constexpr (Pm == 8) {
        const uint4 a = *reinterpret_cast<const uint4*>(base + lane * 16), b = *reinterpret_cast<const uint4*>(base + 512 + lane * 16);
        mw[0] = a.x; mw[1] = a.y; mw[2] = a.z; mw[3] = a.w; mw[4] = b.x; mw[5] = b.y; mw[6] = b.z; mw[7] = b.w;
    } else if constexpr (Pm == 4) {
        const uint4 a = *reinterpret_cast<const uint4*>(base + lane * 16);
        mw[0] = a.x; mw[1] = a.y; mw[2] = a.z; mw[3] = a.w;
    } else {
        const uint2 a = *reinterpret_cast<const uint2*>(base + lane * 8);
        mw[0] = a.x; mw[1] = a.y;
    }
    if constexpr (Pe == 1) {
        ew[0] = *reinterpret_cast<const uint32_t*>(base + 128 * Pm + lane * 4);
    } else if constexpr (Pe == 2) {
        const uint2 a = *reinterpret_cast<const uint2*>(base + 128 * Pm + lane * 8);
        ew[0] = a.x; ew[1] = a.y;
    }
}

// 4-bit fields in "two-offset form": value = offset + q with offset 1024 (even pair slots) or 64 (odd pair slots), i.e. the
// bare (w & mask) | magic -- 4 LOP3 + 1 SHF per 8 weights and nothing else.  The offsets and the zero point are removed per
// group AFTER the tensor core:  sum_k a_k (q_k - z) = D - (S1 + z * S0),  S1 = sum_k a_k * offset_k,  S0 = sum_k a_k;  S1 and
// S0 do not depend on the output column, the warpgroup computes them once per group from the staged activations.
// Products (offset + q) * a are exact in the tensor core and fp32 accumulation sees operands < 2^11 |a|.
__device__ __forceinline__ void tc_dequant4(const uint32_t* mw, uint32_t* A) {
    const uint32_t m0 = 0x000f000fu, g0 = 0x64006400u, m1 = 0x00f000f0u, g1 = 0x54005400u;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
        const uint32_t x = mw[w], y = x >> 8;
        A[w * 4 + 0] = and_or(x, m0, g0);
        A[w * 4 + 1] = and_or(x, m1, g1);
        A[w * 4 + 2] = and_or(y, m0, g0);
        A[w * 4 + 3] = and_or(y, m1, g1);
    }
}
// unpack slab i of this warp's block stage (contiguous at sp) into this thread's row of an A tile (a_row = tile + n * 16)
template <int BITS>
__device__ __forceinline__ void tc_dequant_slab(const uint8_t* sp, int i, int lane, uint8_t* a_row) {
    uint32_t mw[8], ew[2], A[16];
    tc_load_words<BITS>(sp + i * block_bytes(BITS), lane, mw, ew);
    if constexpr (BITS == 4) tc_dequant4(mw, A);
    else dequant_block_exl2<BITS>(mw, ew, A);
#pragma unroll
    for (int kb = 0; kb < 4; ++kb)
        *reinterpret_cast<uint4*>(a_row + kb * TC_A_PLANE) = make_uint4(A[4 * kb], A[4 * kb + 1], A[4 * kb + 2], A[4 * kb + 3]);
}

// ---- activation prep: RMSNorm + q_perm gather + core-matrix layout, once per launch -------------------------------------
// xp[mat][k'/8][tok 0..TW-1][k'%8] = half(x[tok][perm_mat[k']] * w[perm] * rstd[tok])   (rows tok >= M are zero)
// One CTA per token slot (TW CTAs).  The GEMV CTAs then fetch their k-range with ONE bulk copy -- no per-CTA gather.
struct PrepParams {
    const half* x;          // [M][ldx]
    int ldx, M, K, num_mats;
    int tw;                 // token slots of the layout (the launch's tile width)
    const half* norm_w;     // or NULL
    float norm_eps;
    const uint16_t* perm[GEMV_MAX_MATS];
    half* xp[GEMV_MAX_MATS];
};
__global__ void __launch_bounds__(1024) tc_prep_kernel(const __grid_constant__ PrepParams P) {
    griddep_launch_dependents();
    griddep_wait();
    const int tok = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    __shared__ float part[32];
    float rstd = 1.f;
    const bool live = tok < P.M;
    const half* xr = P.x + (size_t)tok * P.ldx;
    if (live && P.norm_w) {            // cuda/rms_norm.cu:55-111: clamp, fp32 sum of squares, rsqrt(mean + eps)
        float sum = 0.f;
        for (int k = tid * 8; k < P.K; k += 1024 * 8) {
            const uint4 v4 = *reinterpret_cast<const uint4*>(xr + k);
            const half2* h2 = reinterpret_cast<const half2*>(&v4);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                float f0 = fmaxf(-65504.f, fminf(__low2float(h2[i]), 65504.f));
                float f1 = fmaxf(-65504.f, fminf(__high2float(h2[i]), 65504.f));
                sum = fmaf(f0, f0, sum);
                sum = fmaf(f1, f1, sum);
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        if (lane == 0) part[warp] = sum;
        __syncthreads();
        float t = (lane < 32) ? part[lane] : 0.f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        rstd = rsqrtf(t * (1.0f / (float)P.K) + P.norm_eps);
    }
    for (int mi = 0; mi < P.num_mats; ++mi) {
        const uint16_t* perm = P.perm[mi];
        half* dst = P.xp[mi];
        for (int kp = tid; kp < P.K; kp += 1024) {
            half v = __float2half(0.f);
            if (live) {
                const int src = perm ? (int)__ldg(perm + kp) : kp;
                v = xr[src];
                if (P.norm_w) {
                    float xf = fmaxf(-65504.f, fminf(__half2float(v), 65504.f));
                    v = __float2half_rn(xf * __half2float(__ldg(P.norm_w + src)) * rstd);
                }
            }
            dst[(size_t)(kp >> 3) * (P.tw * 8) + tok * 8 + (kp & 7)] = v;
        }
    }
}

template <int MT>   // MT = 1 (decode) or 8 tokens per pass on the 8-wide tile; 32 or 64 on the wide tiles
__global__ void __launch_bounds__(TC_THREADS, MT <= GEMV_MTOK ? 2 : 1) gemm_tc_kernel(const __grid_constant__ GemvParams P) {
    constexpr int TW = tc_tile(MT), ACT_STAGE = tc_act_stage(TW), RED = tc_red_floats(TW), NF = TW / 2;
    extern __shared__ __align__(1024) uint8_t smem[];
    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);         // provably warp-uniform
    const int wg = warp >> 2;                                       // the warpgroup this warp belongs to
    const int wq = warp & 3, tidw = tid & 127;                      // warp in the WG; thread = weight column during the unpack

    griddep_launch_dependents();
    EXL2B_STAMP(P, 0);

    // shared memory: [barriers][misc][WG totals][fp16 tile][ssq][S1/S0] | [2 activation rings] | [2 x 2 A tiles] | [8 weight rings]
    // (wide tiles: [WG totals][fp16 tile] overlay the pipeline area from the activation rings on, tc_comb_overlaid)
    const uint32_t smem0 = smem_addr(smem);
    const int stage_bytes = P.tc_stage_bytes, NS = P.tc_stages;
    const uint32_t wbar = smem0 + warp * TC_MAX_STAGES * 8;                                   // my weight stages
    const uint32_t abar = smem0 + (TC_WARPS * TC_MAX_STAGES + wg * TC_MAX_STAGES) * 8;          // my WG's activation stages
    uint8_t* misc = smem + TC_SMEM_BARS;
    int* flag_s = reinterpret_cast<int*>(misc + 64);
    float* rstd_s = reinterpret_cast<float*>(misc + (TW > GEMV_MTOK ? 128 : 16));   // [TW] deferred RMSNorm factors
    uint8_t* const after_misc = misc + tc_misc_bytes(TW);
    float* comb_s = reinterpret_cast<float*>(tc_comb_overlaid(TW) ? smem + P.tc_act_off : after_misc);   // [2 WG][TW][128] totals
    half* tile_s = reinterpret_cast<half*>(comb_s + 2 * TW * 128);            // [TW][128] fp16 outputs (RoPE partner exchange)
    float* ssq_s = reinterpret_cast<float*>(tc_comb_overlaid(TW) ? after_misc : reinterpret_cast<uint8_t*>(tile_s + TW * 128));
    float* corr_s = ssq_s + 4 * TW;                                           // [4][TW] ssq | [parity][WG][warp][S1[TW] | S0[TW]]
    const uint32_t act_ring = smem0 + P.tc_act_off + wg * NS * ACT_STAGE;
    const int a_off = P.tc_act_off + 2 * NS * ACT_STAGE;
    const uint32_t a_tiles = smem0 + a_off + wg * TC_A_BUFS * TC_A_BYTES;
    uint8_t* a_rows = smem + a_off + wg * TC_A_BUFS * TC_A_BYTES + tidw * 16;
    const int ring_off = a_off + 2 * TC_A_BUFS * TC_A_BYTES;
    uint8_t* ring_p = smem + ring_off + warp * NS * stage_bytes;
    const uint32_t ring = smem0 + ring_off + warp * NS * stage_bytes;
    const int M = P.M, KS = P.KS;

    // ---- one-time setup: barriers ----
    if (lane == 0) {
        for (int st = 0; st < NS; ++st) mbar_init(wbar + 8 * st, 1);
        if (wq == 0)
            for (int st = 0; st < NS; ++st) mbar_init(abar + 8 * st, 1);
        mbar_fence_init();
    }
    __syncwarp();
    // (a warp's weight barriers are used by that warp alone: it may start fetching right away; the CTA-wide barrier that
    //  publishes the shared barriers comes after the first requests are in flight)
    bool setup_done = false;

    const unsigned U = (unsigned)P.total_units, G = gridDim.x;
    const int u0 = (int)((unsigned)blockIdx.x * U / G), u1 = (int)(((unsigned)blockIdx.x + 1u) * U / G);

    uint32_t wphase = 0, aphase = 0;     // parity bits per barrier
    uint32_t gpar = 0;                   // parity of the S1 / S0 buffer of the current group
    bool waited = false;
    auto after_wait = [&]() {       // first point where the previous kernel's output may be read
        if (P.ex.sumsq_in) {        // warp w: 1/rms of tokens w, w + 8, ..., strips summed in a fixed order
#pragma unroll 1
            for (int m = warp; m < TW; m += TC_WARPS) {
                float sum = 0.f;
                for (int sidx = lane; sidx < P.ex.sumsq_in_strips; sidx += 32) sum += __ldcg(P.ex.sumsq_in + sidx * TW + m);
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
                if (lane == 0) rstd_s[m] = rsqrtf(sum / (float)(KS * SLAB_K) + P.ex.sumsq_eps);
            }
        }
    };

    int u = u0;
    while (u < u1) {
        int mi = 0;
        while (mi + 1 < P.num_mats && u >= P.mat[mi + 1].unit_begin) ++mi;
        const GemvMat& mt = P.mat[mi];
        const QMatView& w = mt.w;
        const int local = u - mt.unit_begin;
        const int strip = local / KS, ks_a = local - strip * KS;
        const int seg = min(KS - ks_a, u1 - u);
        // snap the slab range to group boundaries (every CTA applies the same rule, so ranges still tile the strip);
        // WG0 takes the first half of the range's groups, WG1 the second: two contiguous streams per CTA
        const int ks0 = tc_group_start(w, ks_a), ks1 = tc_group_start(w, ks_a + seg);
        const int ksm = tc_group_start(w, ks0 + ((ks1 - ks0 + 1) >> 1));
        const int my0 = wg ? ksm : ks0, my1 = wg ? ks1 : ksm;
        const int n_col = strip * 128 + tidw;                                  // this thread's column in the epilogue
        const uint8_t* gsrc = reinterpret_cast<const uint8_t*>(w.packed) + (size_t)strip * w.strip_bytes + (size_t)wq * w.blk_stream_bytes;
        const uint8_t* asrc = reinterpret_cast<const uint8_t*>(mt.xp);
        const int nreg = w.num_regions;
        // accumulator fragment of wgmma m64n8: row 16 wq + lane / 4 (+ 8) of each M tile, tokens 2 (lane % 4) (+ 1).  Fragment
        // column j (j = 2 * tile + half) is strip column cb + 8 * cofs[j]
        const int cb = strip * 128 + 16 * wq + (lane >> 2), t0 = 2 * (lane & 3);
        // per-matrix fields used in the loops below, pinned in registers (indexed kernel-parameter reads are slow and the
        // compiler would otherwise re-read them every group)
        const bool gptq = w.is_gptq != 0;
        const uint32_t* sc_w = (gptq ? w.qzeros : w.q_scale) + (cb >> 3);      // nibble word of column cb, group 0
        const half* sc_h = gptq ? w.gptq_scales + cb : w.q_scale_max;
        int n8 = w.N >> 3;
        asm volatile("" : "+l"(sc_w));
        asm volatile("" : "+l"(sc_h));
        asm volatile("" : "+r"(n8));
        const int nib_sh = (cb & 7) * 4;
        bool live[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) live[j] = cb + 8 * ((j & 1) + 8 * (j >> 1)) < w.N;

        // Group cursors: position + the current region's parameters in registers, so that stepping to the next group
        // is a handful of integer ops; the kernel-parameter region table is only read when a region boundary is crossed.
        //   C: the group being unpacked;   F: the next group to request (weights + activations), NS groups ahead
        int c_ks = my0, c_r = tc_region_of(w, min(my0, KS - 1));
        int c_bits = w.reg[c_r].bits, c_spg = 1 << w.reg[c_r].spg_log2, c_end = tc_region_end(w, c_r);
        int c_grp = w.reg[c_r].group_base + ((my0 - w.reg[c_r].ks_begin) >> w.reg[c_r].spg_log2);
        int f_ks = c_ks, f_r = c_r, f_bits = c_bits, f_spg = c_spg, f_end = c_end;
        uint32_t f_off = w.reg[c_r].off_base + (uint32_t)(my0 - w.reg[c_r].ks_begin) * (uint32_t)block_bytes(c_bits);
        int f_stage = 0, cstage = 0;

        // request group F's weights (every warp: its own block) and, optionally, its activations (the WG's first warp)
        auto issue = [&](bool weights, bool acts) {
            const int ns = min(f_spg, f_end - f_ks);
            const uint32_t wbytes = (uint32_t)ns * (uint32_t)block_bytes(f_bits);
            if (elect_one()) {
                if (weights) {
                    mbar_arrive_expect_tx(wbar + 8 * f_stage, wbytes);
                    bulk_copy_g2s(ring + f_stage * stage_bytes, gsrc + f_off, wbytes, wbar + 8 * f_stage);
                }
                if (acts && wq == 0) {
                    mbar_arrive_expect_tx(abar + 8 * f_stage, (uint32_t)ns * SLAB_K * TW * 2);
                    bulk_copy_g2s(act_ring + f_stage * ACT_STAGE, asrc + (size_t)f_ks * SLAB_K * TW * 2, (uint32_t)ns * SLAB_K * TW * 2,
                                  abar + 8 * f_stage);
                }
            }
            f_ks += ns;
            f_off += wbytes;
            f_stage = (f_stage + 1 == NS) ? 0 : f_stage + 1;
            if (f_ks >= f_end && f_r + 1 < nreg) {
                ++f_r;
                f_bits = w.reg[f_r].bits;
                f_spg = 1 << w.reg[f_r].spg_log2;
                f_end = tc_region_end(w, f_r);
                f_off = w.reg[f_r].off_base;
            }
        };
        // prologue: the first NS groups' weights (they never depend on a previous kernel); their activations follow after
        // griddepcontrol.wait, requested by re-walking the same groups with a scratch copy of the cursor
        int primed = 0;
#pragma unroll 1
        for (; primed < NS && f_ks < my1; ++primed) issue(true, false);
        if (!setup_done) {
            setup_done = true;
            __syncthreads();
        }
        EXL2B_STAMP(P, 1);

        // everything above depended only on the weights; from here on the previous kernel's output is needed
        if (!waited) {
            griddep_wait();
            waited = true;
            after_wait();
            EXL2B_STAMP(P, 2);
        }
        if (wq == 0) {            // the activations of the groups primed above (same walk, scratch cursor)
            int t_ks = my0, t_r = c_r, t_spg = c_spg, t_end = c_end;
            for (int st = 0; st < primed; ++st) {
                const int tn = min(t_spg, t_end - t_ks);
                if (elect_one()) {
                    mbar_arrive_expect_tx(abar + 8 * st, (uint32_t)tn * SLAB_K * TW * 2);
                    bulk_copy_g2s(act_ring + st * ACT_STAGE, asrc + (size_t)t_ks * SLAB_K * TW * 2, (uint32_t)tn * SLAB_K * TW * 2, abar + 8 * st);
                }
                t_ks += tn;
                if (t_ks >= t_end && t_r + 1 < nreg) {
                    ++t_r;
                    t_spg = 1 << w.reg[t_r].spg_log2;
                    t_end = tc_region_end(w, t_r);
                }
            }
        }

        // ---- the pipeline of a warpgroup, one group per iteration ----
        float frag[2][NF], acc[2][NF];   // running totals / the current group's sums, fragment order (wgmma_tile): [M tile][i]
#pragma unroll
        for (int t = 0; t < 2; ++t)
#pragma unroll
            for (int i = 0; i < NF; ++i) frag[t][i] = acc[t][i] = 0.f;
        while (c_ks < my1) {
            const int bits = c_bits;
            const int ns = min(c_spg, c_end - c_ks);
            const int grp = c_grp;

            // (a) this group's scales for my four fragment columns: requested now, used after the group's MMAs
            uint32_t sw[4];
            half sh[4];
            half smax = __float2half(0.f);
            if (!gptq) smax = __ldg(sc_h + grp);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int cofs = (j & 1) + 8 * (j >> 1);           // in nibble words (8 columns)
                sw[j] = live[j] ? __ldg(sc_w + (size_t)grp * n8 + cofs) : 0u;
                sh[j] = (gptq && live[j]) ? __ldg(sc_h + (size_t)grp * (n8 * 8) + 8 * cofs) : __float2half(0.f);
            }

            // (b) my block's slabs and the WG's activations of this group have landed
            mbar_wait(wbar + 8 * cstage, (wphase >> cstage) & 1u);
            wphase ^= 1u << cstage;
            mbar_wait(abar + 8 * cstage, (aphase >> cstage) & 1u);
            aphase ^= 1u << cstage;
            const uint8_t* sp = ring_p + cstage * stage_bytes;
            const uint32_t actb = act_ring + cstage * ACT_STAGE;

            // (c) 4-bit offset form: this warp's share of S1 / S0 (8-k rows 4 wq .. 4 wq + 3 of the group); published to the
            //     other warps by the slab barriers below, read after them; 8 tokens per round
            if (bits == 4) {
                const int row = wq * 4 + (lane >> 3);
                float* cw = corr_s + ((gpar * 2 + wg) * 4 + wq) * 2 * TW;
#pragma unroll
                for (int tb = 0; tb < TW; tb += 8) {
                    const int t = tb + (lane & 7);
                    float s1 = 0.f, s0 = 0.f;
                    if (row < ns * 4) {
                        const uint4 v = *reinterpret_cast<const uint4*>(smem + P.tc_act_off + (wg * NS + cstage) * ACT_STAGE + row * (TW * 16) + t * 16);
                        const float2 f0 = __half22float2(*reinterpret_cast<const half2*>(&v.x)), f1 = __half22float2(*reinterpret_cast<const half2*>(&v.y));
                        const float2 f2 = __half22float2(*reinterpret_cast<const half2*>(&v.z)), f3 = __half22float2(*reinterpret_cast<const half2*>(&v.w));
                        const float e = (f0.x + f0.y) + (f2.x + f2.y), o = (f1.x + f1.y) + (f3.x + f3.y);   // even / odd pair slots
                        s1 = fmaf(1024.f, e, 64.f * o);
                        s0 = e + o;
                    }
                    s1 += __shfl_xor_sync(0xffffffffu, s1, 8);
                    s0 += __shfl_xor_sync(0xffffffffu, s0, 8);
                    s1 += __shfl_xor_sync(0xffffffffu, s1, 16);
                    s0 += __shfl_xor_sync(0xffffffffu, s0, 16);
                    if (lane < 8) {
                        cw[t] = s1;
                        cw[TW + t] = s0;
                    }
                }
            }

            // (d) unpack slab by slab into the A tiles; the WG issues the slab's MMAs as soon as all 128 rows are stored.  The
            //     first MMA of a group overwrites the accumulator (which only wgmma writes, so the MMAs stay asynchronous)
#pragma unroll 1
            for (int i = 0; i < ns; ++i) {
                const int ab = i & 1;
                if (i >= TC_A_BUFS) wg_wait<TC_A_BUFS - 1>();         // the MMAs that read this tile two slabs ago have retired
                uint8_t* arow = a_rows + ab * TC_A_BYTES;
                switch (bits) {
                    case 4: tc_dequant_slab<4>(sp, i, lane, arow); break;
                    case 5: tc_dequant_slab<5>(sp, i, lane, arow); break;
                    case 3: tc_dequant_slab<3>(sp, i, lane, arow); break;
                    case 6: tc_dequant_slab<6>(sp, i, lane, arow); break;
                    case 2: tc_dequant_slab<2>(sp, i, lane, arow); break;
                    default: tc_dequant_slab<8>(sp, i, lane, arow); break;
                }
                fence_proxy_async_smem();
                bar_sync(1 + wg, 128);
                wg_fence();
                // B: plane kb (k 8kb .. 8kb+7) of the slab at kb * TW * 16, token t at t * 16 within it
                const uint32_t at = a_tiles + ab * TC_A_BYTES, bt = actb + i * (SLAB_K / 8) * (TW * 16);
#pragma unroll
                for (int s = 0; s < 2; ++s) {
#pragma unroll
                    for (int t = 0; t < 2; ++t)
                        wgmma_tile(acc[t], make_desc(at + s * 2 * TC_A_PLANE + t * 64 * 16, TC_A_PLANE, 128),
                                   make_desc(bt + s * 2 * (TW * 16), TW * 16, TW > 8 ? 128 : 0), (i | s) ? 1u : 0u);
                }
                wg_commit();
            }
            wg_wait<0>();
            wg_fence_acc(acc[0]);
            wg_fence_acc(acc[1]);

            // (e) scale the group's sums into the running totals: sum_k a_k w_k = scale * (D - (S1 + z * S0)) per column
            float scl[4], zfs[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int nib = (int)((sw[j] >> nib_sh) & 15u);
                float scale, zf = 8.f;
                if (!gptq) {
                    scale = __half2float(__hmul(__int2half_rn((nib + 1) * (nib + 1)), smax));    // qdq_util.cuh:24-30
                } else {
                    scale = __half2float(sh[j]);
                    zf = (float)(nib + 1);                                                          // q_gemm_kernel_gptq.cuh:167-172
                }
                scl[j] = live[j] ? scale : 0.f;
                zfs[j] = zf;
            }
#pragma unroll
            for (int nb = 0; nb < TW / 8; ++nb) {          // tokens 8 nb + t0, + 1
                float c1[2] = {0.f, 0.f}, c0[2] = {0.f, 0.f};
                if (bits == 4) {
                    const float* cr = corr_s + (gpar * 2 + wg) * 4 * 2 * TW + 8 * nb + t0;
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        c1[e] = (cr[e] + cr[2 * TW + e]) + (cr[4 * TW + e] + cr[6 * TW + e]);
                        c0[e] = (cr[TW + e] + cr[3 * TW + e]) + (cr[5 * TW + e] + cr[7 * TW + e]);
                    }
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    float* f = &frag[j >> 1][4 * nb + (j & 1) * 2];
                    const float* d = &acc[j >> 1][4 * nb + (j & 1) * 2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) f[e] = fmaf(scl[j], d[e] - fmaf(zfs[j], c0[e], c1[e]), f[e]);
                }
            }

            // (f) the group's MMAs have retired: both of its stages are free for the next request
            if (f_ks < my1) issue(true, true);
            gpar ^= 1u;
            cstage = (cstage + 1 == NS) ? 0 : cstage + 1;
            c_ks += ns;
            ++c_grp;
            if (c_ks >= c_end && c_r + 1 < nreg) {
                ++c_r;
                c_bits = w.reg[c_r].bits;
                c_spg = 1 << w.reg[c_r].spg_log2;
                c_end = tc_region_end(w, c_r);
                c_grp = w.reg[c_r].group_base;
            }
        }
        if (!waited) {        // a CTA whose snapped range is empty still takes part in the fix-up below
            griddep_wait();
            waited = true;
            after_wait();
        }
        EXL2B_STAMP(P, 4);

        // the finishing CTA's scatter needs, per consumer, this column's destination row and RMSNorm weight: request them now, so
        // that the loads ride under the combine / split-K hand-off below instead of sitting on the tail of the launch
        int skp[GEMV_MAX_MATS];
        half ssc[GEMV_MAX_MATS];
        half resid0 = __float2half(0.f);            // decode (one row): the residual element this column adds to, same idea
        if constexpr (MT == 1) {
            if (wg == 0 && P.epilogue == EPI_STORE && !mt.clear && n_col < w.N) resid0 = mt.c[n_col];
        }
        {
            const bool col_any = n_col < ((P.epilogue != EPI_STORE) ? P.mat[0].w.N : w.N);
#pragma unroll
            for (int t = 0; t < GEMV_MAX_MATS; ++t) {
                skp[t] = n_col;
                ssc[t] = __float2half(1.f);
                if (wg == 0 && t < P.ex.num_scat && col_any) {
                    if (P.ex.scat[t].invperm) skp[t] = (int)__ldg(P.ex.scat[t].invperm + n_col);
                    if (P.ex.scat[t].scale) ssc[t] = __ldg(P.ex.scat[t].scale + n_col);
                }
            }
        }

        // ---- both warpgroups' fragments -> column order (thread = column), then the split-K / epilogue logic ----
        __syncthreads();
        {
            float* cw = comb_s + wg * (TW * 128);
#pragma unroll
            for (int nb = 0; nb < TW / 8; ++nb)
#pragma unroll
                for (int j = 0; j < 4; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e)
                        if (8 * nb + t0 + e < MT)
                            cw[(8 * nb + t0 + e) * 128 + (cb - strip * 128) + 8 * ((j & 1) + 8 * (j >> 1))] = frag[j >> 1][4 * nb + (j & 1) * 2 + e];
        }
        __syncthreads();
        // this CTA's sum of row m over both warpgroups
        auto tot = [&](int m) { return comb_s[m * 128 + tidw] + comb_s[TW * 128 + m * 128 + tidw]; };

        const int gs = mt.strip_begin + strip;
        const unsigned sb = (unsigned)mt.unit_begin + (unsigned)strip * KS;
        const int first_cta = tc_cta_of_unit(sb, G, U), last_cta = tc_cta_of_unit(sb + KS - 1, G, U);
        const int nc = last_cta - first_cta + 1, jc = (int)blockIdx.x - first_cta;
        const bool paired = P.epilogue != EPI_STORE;
        const bool has_rstd = P.ex.sumsq_in != nullptr;
        const bool alone = nc == 1 && !paired;     // this CTA holds the strip's complete sums
        bool finisher = alone;
        if (!alone) {
            float* wsp = P.ws + ((size_t)gs * P.maxc + jc) * RED;
            if (wg == 0) {
#pragma unroll (MT <= GEMV_MTOK ? MT : 4)
                for (int m = 0; m < MT; ++m) __stcg(wsp + m * 128 + tidw, tot(m));
            }
            __syncthreads();             // every partial of this CTA is written (CTA-scope happens-before to thread 0)
            int expected = nc, cidx = gs;
            if (paired) {
                const GemvMat& other = P.mat[1 - mi];
                const unsigned ob = (unsigned)other.unit_begin + (unsigned)strip * KS;
                expected += tc_cta_of_unit(ob + KS - 1, G, U) - tc_cta_of_unit(ob, G, U) + 1;
                cidx = P.mat[0].strip_begin + strip;
            }
            if (tid == 0) {              // release our partials / acquire everybody else's: one acq_rel RMW at GPU scope
                unsigned int old;
                asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], %2;" : "=r"(old) : "l"(P.counters + cidx), "r"(1u) : "memory");
                *flag_s = (old == (unsigned int)(expected - 1)) ? 1 : 0;
            }
            __syncthreads();
            if (*flag_s) {
                finisher = true;
                if (tid == 0) P.counters[cidx] = 0u;
            }
        }

        // ---- the finishing CTA's first warpgroup turns the sums into outputs (thread = column), row by row ----
        if (finisher && wg == 0) {
            const GemvMat& mo = paired ? P.mat[0] : mt;         // where the result goes
            const bool col_ok = n_col < mo.w.N;
            // the strip's complete fp32 sums of a row, from the contributors' partials in a fixed order (vu: the up projection)
            const float* bg = P.ws + (size_t)gs * P.maxc * RED;
            const float* bu = bg;
            int ncg = nc, ncu = 0;
            if (paired) {
                const GemvMat& mg = P.mat[0];
                const GemvMat& mu = P.mat[1];
                const unsigned gb = (unsigned)mg.unit_begin + (unsigned)strip * KS;
                const unsigned ub = (unsigned)mu.unit_begin + (unsigned)strip * KS;
                ncg = tc_cta_of_unit(gb + KS - 1, G, U) - tc_cta_of_unit(gb, G, U) + 1;
                ncu = tc_cta_of_unit(ub + KS - 1, G, U) - tc_cta_of_unit(ub, G, U) + 1;
                bg = P.ws + (size_t)(mg.strip_begin + strip) * P.maxc * RED;
                bu = P.ws + (size_t)(mu.strip_begin + strip) * P.maxc * RED;
            }
            // (1) every row's fp16 value into tile_s: bias, residual or act(gate) * up
#pragma unroll (MT <= GEMV_MTOK ? MT : 4)
            for (int m = 0; m < MT; ++m) {
                float vg = 0.f, vu = 0.f;
                if (alone) {
                    vg = tot(m);
                } else {
                    for (int j = 0; j < ncg; ++j) vg += __ldcg(bg + (size_t)j * RED + m * 128 + tidw);
                    for (int j = 0; j < ncu; ++j) vu += __ldcg(bu + (size_t)j * RED + m * 128 + tidw);
                }
                const float rs = has_rstd ? rstd_s[m] : 1.f;
                half hv;
                if (paired) {
                    vg *= rs;
                    vu *= rs;
                    if (col_ok && P.mat[0].w.bias) vg += __half2float(P.mat[0].w.bias[n_col]);
                    if (col_ok && P.mat[1].w.bias) vu += __half2float(P.mat[1].w.bias[n_col]);
                    const half hg = __float2half_rn(vg), hu = __float2half_rn(vu);           // q_mlp.cu:187-196 roundings
                    const half act = (P.epilogue == EPI_GELU_MUL) ? tc_gelu_h(hg) : tc_silu_h(hg);
                    hv = __hmul(act, hu);
                } else {
                    float v = vg * rs;
                    if (col_ok && m < M) {
                        if (w.bias) v += __half2float(w.bias[n_col]);
                        if (!mt.clear) v += __half2float(MT == 1 ? resid0 : mt.c[(size_t)m * mt.ldc + n_col]);
                    }
                    hv = __float2half_rn(v);
                }
                tile_s[m * 128 + tidw] = hv;
            }
            // (2) RoPE (partner column through tile_s), store, scatter into the consumers, sums of squares
            const bool rope = (P.ex.rope.mask >> mi) & 1u;
            if (rope) bar_sync(3, 128);
            const RopeFuse& R = P.ex.rope;
            const int d = tidw % max(R.head_dim, 1), S = R.sincos_size, hd2 = S >> 1;
#pragma unroll (MT <= GEMV_MTOK ? MT : 4)
            for (int m = 0; m < MT; ++m) {
                half hv = tile_s[m * 128 + tidw];
                if (rope && m < M && d < S) {
                    const int row = P.row0 + m, bb = row / R.q_len, tt = row - bb * R.q_len;
                    int base = R.past_len;
                    if (base == -1) base = max(R.past_lens[bb], 0);
                    else if (R.past_lens) base += R.past_lens[bb];
                    const size_t sr = (size_t)max(base + tt, 0) * S;
                    if (R.neox) {
                        if (d < hd2) {
                            const half c = R.cos[sr + d], sn = R.sin[sr + d];
                            hv = __hfma(hv, c, __hmul(tile_s[m * 128 + tidw + hd2], __hneg(sn)));
                        } else {
                            const half c = R.cos[sr + d - hd2], sn = R.sin[sr + d - hd2];
                            hv = __hfma(hv, c, __hmul(tile_s[m * 128 + tidw - hd2], sn));
                        }
                    } else {
                        const half c = R.cos[sr + d], sn = R.sin[sr + d];
                        if ((d & 1) == 0) hv = __hfma(tile_s[m * 128 + tidw + 1], __hneg(sn), __hmul(hv, c));
                        else hv = __hfma(tile_s[m * 128 + tidw - 1], sn, __hmul(hv, c));
                    }
                }
                float ssq = 0.f;
                if (col_ok && m < M) {
                    mo.c[(size_t)m * mo.ldc + n_col] = hv;
                    const float f = fmaxf(-65504.f, fminf(__half2float(hv), 65504.f));
                    ssq = f * f;
#pragma unroll
                    for (int t = 0; t < GEMV_MAX_MATS; ++t) {
                        if (t < P.ex.num_scat) {
                            const ScatterTarget& T = P.ex.scat[t];
                            const int kp = skp[t];
                            const half o = T.scale ? __float2half_rn(f * __half2float(ssc[t])) : hv;
                            T.xp[(size_t)(kp >> 3) * (TW * 8) + m * 8 + (kp & 7)] = o;
                        }
                    }
                }
                if (P.ex.sumsq_out) {
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) ssq += __shfl_xor_sync(0xffffffffu, ssq, o);
                    if (lane == 0) ssq_s[wq * TW + m] = ssq;
                }
            }
            if (P.ex.sumsq_out) {        // per-strip sum of squares of the stored rows, fixed reduction order
                bar_sync(3, 128);
                if (tidw < TW) {
                    const float t4 = (ssq_s[tidw] + ssq_s[TW + tidw]) + (ssq_s[2 * TW + tidw] + ssq_s[3 * TW + tidw]);
                    P.ex.sumsq_out[(size_t)strip * TW + tidw] = (tidw < MT) ? t4 : 0.f;
                }
            }
        }
        // the wide tiles' combine buffer overlays the rings the next segment's bulk copies write: order its generic-proxy
        // accesses before them
        if constexpr (tc_comb_overlaid(TW)) fence_proxy_async_smem();
        __syncthreads();
        EXL2B_STAMP(P, 5);
        u += seg;
    }

    if (P.dbg && tid == 0) atomicMax(P.dbg + 7, globaltimer());
}

// ---- host launcher -----------------------------------------------------------------------------------------------------

int gemv_workspace(int device, cudaStream_t stream, bool wide, float** ws, unsigned int** counters, size_t* ws_bytes, int* n_counters,
                   half** xp, size_t* xp_bytes);

int gemm_tc_launch(int device, cudaStream_t stream, GemvMat* mats, int nm, int M, const half* norm_w, float norm_eps, int epilogue,
                   const GemvExtras* ex) {
    EXL2B_REQUIRE(nm >= 1 && nm <= GEMV_MAX_MATS, "bad matrix count %d", nm);
    if (M <= 0) return 0;
    // a launch with fused extras runs its rows in one pass, on the narrowest tile that holds them; without, in 8-row passes
    if (ex) EXL2B_REQUIRE(M <= GEMV_MAX_CHAIN_ROWS, "fused epilogue extras need a single pass of at most %d rows (rows %d)",
                          GEMV_MAX_CHAIN_ROWS, M);
    const bool wide = ex && M > GEMV_MTOK;
    const int tw = wide ? tc_tile(M) : GEMV_MTOK, pass = wide ? M : GEMV_MTOK;
    float* ws = nullptr;
    unsigned int* counters = nullptr;
    size_t ws_bytes = 0, xp_bytes = 0;
    int n_counters = 0;
    half* xp_scratch = nullptr;
    int rc = gemv_workspace(device, stream, wide, &ws, &counters, &ws_bytes, &n_counters, &xp_scratch, &xp_bytes);
    if (rc) return rc;
    static std::atomic<bool> attr_set[64];
    if (!attr_set[device].load()) {
        EXL2B_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_CAP));
        EXL2B_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_CAP));
        EXL2B_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_CAP));
        EXL2B_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_CAP));
        attr_set[device].store(true);
    }

    GemvParams P = {};
    P.num_mats = nm;
    P.KS = mats[0].w.KS;
    const bool prepared = ex && ex->prepared;
    if (ex) {
        P.ex = *ex;
        if (ex->rope.mask) EXL2B_REQUIRE(ex->rope.head_dim > 0 && 128 % ex->rope.head_dim == 0 && ex->rope.sincos_size <= ex->rope.head_dim,
                                         "fused RoPE needs head_dim to divide 128");
        if (ex->sumsq_in) P.ex.sumsq_eps = norm_eps;
    }
    const size_t xp_per_mat = xp_bytes / GEMV_MAX_MATS;
    long long units = 0;
    int strips = 0;
    for (int i = 0; i < nm; ++i) {
        EXL2B_REQUIRE(mats[i].w.layout == LAYOUT_TC, "matrix is not in the default (LAYOUT_TC) layout");
        EXL2B_REQUIRE(mats[i].w.KS == P.KS, "fused matrices must share K");
        EXL2B_REQUIRE(prepared || (mats[i].x == mats[0].x && mats[i].ldx == mats[0].ldx), "fused matrices must share their input");
        P.mat[i] = mats[i];
        P.mat[i].unit_begin = (int)units;
        P.mat[i].strip_begin = strips;
        if (prepared) EXL2B_REQUIRE(mats[i].xp, "prepared launch without an activation buffer");
        else P.mat[i].xp = xp_scratch + (size_t)i * (xp_per_mat / sizeof(half));
        units += (long long)mats[i].w.strips * P.KS;
        strips += mats[i].w.strips;
    }
    if (norm_w && !prepared) EXL2B_REQUIRE(mats[0].w.K % 8 == 0 && mats[0].ldx % 8 == 0, "fused RMSNorm needs K and the row stride to be multiples of 8");
    if (epilogue != EPI_STORE) EXL2B_REQUIRE(nm == 2 && mats[0].w.N == mats[1].w.N, "gate/up epilogue needs two matrices of equal width");
    P.norm_w = norm_w;
    P.norm_eps = norm_eps;
    P.epilogue = epilogue;
    P.ws = ws;
    P.counters = counters;

    // Grid: every strip cut into S equal K-ranges (one segment per CTA) or plain stream-K over all resident slots --
    // whichever has the cheaper slowest CTA under  cost = segments * F + slabs  (F = per-segment fixed cost in slabs).
    // The wide tiles hold one CTA per SM (registers and shared memory).
    extern int g_tc_ctas_per_sm;
    const int ctas_per_sm = wide ? 1 : g_tc_ctas_per_sm;
    const int sms = device_sm_count(device);
    const long long slots = (long long)sms * ctas_per_sm;
    const long long F = 16;
    long long grid_ll = std::min(slots, units);
    {
        const long long L = (units + grid_ll - 1) / grid_ll;
        const long long cost_stream = ((L + P.KS - 1) / P.KS + 1) * F + L;
        if (strips <= slots) {
            // S need not divide KS: CTA i covers units [i*U/G, (i+1)*U/G), every S-th boundary is a strip boundary, the others
            // are snapped to quantisation-group starts by the kernel -- still exactly one segment per CTA
            const int S = (int)std::min<long long>(slots / strips, std::max(1, P.KS / 8));
            const long long cost_aligned = F + (P.KS + S - 1) / S;
            if (cost_aligned <= cost_stream) grid_ll = (long long)strips * S;
        }
    }
    const int grid = (int)std::max(1ll, grid_ll);
    EXL2B_REQUIRE((units + 1) * grid < (1ll << 31), "problem too large for 32-bit unit arithmetic");
    P.total_units = (int)units;
    P.maxc = (int)(((long long)P.KS * grid) / units) + 2;
    EXL2B_REQUIRE(strips <= n_counters, "too many strips for the counter array");
    EXL2B_REQUIRE((size_t)strips * P.maxc * tc_red_floats(tw) * sizeof(float) <= ws_bytes, "split-K workspace too small");

    // stage = the largest group of any matrix of the launch, per 32-column block
    int stage_bytes = 0;
    for (int i = 0; i < nm; ++i)
        for (int r = 0; r < mats[i].w.num_regions; ++r) {
            // a stage's activations are one activation stage (128 k): a larger group would overrun the activation ring
            EXL2B_REQUIRE(mats[i].w.reg[r].spg_log2 <= 2, "quantisation groups above 128 rows are not supported by the wgmma kernel");
            stage_bytes = std::max(stage_bytes, (1 << mats[i].w.reg[r].spg_log2) * block_bytes(mats[i].w.reg[r].bits));
        }
    EXL2B_REQUIRE(stage_bytes > 0 && stage_bytes <= 4096, "quantisation groups above 128 rows are not supported by the wgmma kernel");
    P.tc_stage_bytes = stage_bytes;
    const int header = tc_header_bytes(tw);
    P.tc_act_off = header;
    // as many stages (<= 4) as leave room for the intended number of CTAs per SM (227 KB of shared memory, 1 KB reserved per CTA)
    const size_t smem_budget = std::min<size_t>((size_t)(227 * 1024) / (size_t)std::max(1, ctas_per_sm) - 1024, TC_SMEM_CAP);
    int stages = TC_MAX_STAGES;
    auto smem_for = [&](int st) {
        return (size_t)header + 2 * TC_A_BUFS * TC_A_BYTES + (size_t)st * (2 * tc_act_stage(tw) + (size_t)TC_WARPS * stage_bytes);
    };
    while (stages > 2 && smem_for(stages) > smem_budget) --stages;
    P.tc_stages = stages;
    P.tc_act_bytes = 2 * stages * tc_act_stage(tw);
    const size_t smem_total = smem_for(stages);
    EXL2B_REQUIRE(smem_total <= TC_SMEM_CAP, "shared memory budget exceeded (%zu bytes)", smem_total);
    EXL2B_REQUIRE(!tc_comb_overlaid(tw) || (size_t)tc_comb_bytes(tw) <= smem_total - header, "combine buffer does not fit the pipeline area");
    EXL2B_REQUIRE((size_t)mats[0].w.K * tw * 2 <= xp_per_mat, "K too large for the activation scratch");
    extern unsigned long long* g_dbg;
    extern int g_dbg_cta, g_dbg_slot;
    P.dbg_cta = g_dbg_cta;

    PrepParams Q = {};
    Q.ldx = mats[0].ldx;
    Q.K = mats[0].w.K;
    Q.num_mats = nm;
    Q.tw = tw;
    Q.norm_w = norm_w;
    Q.norm_eps = norm_eps;
    for (int i = 0; i < nm; ++i) {
        Q.perm[i] = mats[i].w.perm;
        Q.xp[i] = const_cast<half*>(P.mat[i].xp);
    }
    for (int m0 = 0; m0 < M; m0 += pass) {
        P.M = std::min(pass, M - m0);
        P.dbg = g_dbg ? g_dbg + 32 * (g_dbg_slot++ % 64) : nullptr;
        for (int i = 0; i < nm; ++i) {
            if (!prepared) P.mat[i].x = mats[i].x + (size_t)m0 * mats[i].ldx;
            P.mat[i].c = mats[i].c + (size_t)m0 * mats[i].ldc;
        }
        P.row0 = m0;
        if (!prepared) {
            Q.x = mats[0].x + (size_t)m0 * mats[0].ldx;
            Q.M = P.M;
            EXL2B_CUDA(launch_pdl_f("tc", tc_prep_kernel, dim3(tw), dim3(1024), 0, stream, Q));
        }
        if (P.M == 1) {
            EXL2B_CUDA(launch_pdl_f("tc", gemm_tc_kernel<1>, dim3(grid), dim3(TC_THREADS), smem_total, stream, P));
        } else if (tw == GEMV_MTOK) {
            EXL2B_CUDA(launch_pdl_f("tc", gemm_tc_kernel<8>, dim3(grid), dim3(TC_THREADS), smem_total, stream, P));
        } else if (tw == 32) {
            EXL2B_CUDA(launch_pdl_f("tc", gemm_tc_kernel<32>, dim3(grid), dim3(TC_THREADS), smem_total, stream, P));
        } else {
            EXL2B_CUDA(launch_pdl_f("tc", gemm_tc_kernel<64>, dim3(grid), dim3(TC_THREADS), smem_total, stream, P));
        }
    }
    return 0;
}

}  // namespace exl2b
