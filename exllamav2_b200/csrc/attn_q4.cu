// Decode attention straight over the Q4 / Q6 / Q8 K/V cache: quantise-and-append the new rows, attend, in ONE kernel.
//
// The reference runs, per layer and per step (exllamav2/attn.py:560-613, cache.py:472-556):
//     q_to_fp16_kv over the WHOLE live cache -> flash_attn_with_kvcache on the fp16 temp -> fp16_to_q_kv of the new rows
// i.e. it expands every cached nibble to fp16 in HBM and reads it back.  Here the cache is consumed as stored
// (0.5 B + 1/16 B per value):
//   * the cache holds y = H32 x per 64-value unit (unnormalised Hadamard on the even / odd interleaved 32-vectors,
//     cache_q.cuh), quantised to 4 bits with an fp16 scale per 32 consecutive values.  H is symmetric and H H = 32 I, so
//         q . x = (H q) . y / 32            sum_s p_s x_s = H (sum_s p_s y_s) / 32
//     the query is rotated ONCE, scores and the P V sum are formed on the stored (rotated) values, and the output is
//     rotated back ONCE -- no per-position butterflies.
//   * the kernel is templated on the element widths of keys (KB) and values (VB): (4, 4) is the Q4 cache, (8, 4) Q6 and
//     (8, 8) Q8 (kvcache.cu).  An 8-bit row holds value e of a 32-value block at byte e, one fp16 scale per block as in Q4.
//   * the q_len new K/V rows are quantised with exactly the arithmetic of fp16_to_q_kv (kvcache.cu pack_unit_q4, same
//     bits as the reference) and written to the paged cache by one designated CTA per kv head.  The step that appends
//     them attends them UNQUANTISED (fp16 values, rotated in fp32), exactly like the reference, where
//     flash_attn_with_kvcache sees the fp16 rows and the cache only quantises them afterwards (attn.py:602-621).
// One CTA per (head, sequence); decode regime (q_len <= 8).
#include <algorithm>

#include "gemv_i8.cuh"
#include "qmatrix.cuh"

namespace exl2b {

extern unsigned long long* g_dbg;
extern int g_dbg_cta, g_dbg_slot;

constexpr int AQ_THREADS = 256;
constexpr int AQ_WARPS = 8;
constexpr int AQ_MAX_QLEN = 8;

struct AttnQ4Params {
    const half* q;          // [batch, q_len, H, hd]     (RoPE already applied)
    const half* k_new;      // [batch, q_len, KVH, hd]
    const half* v_new;
    uint8_t* k_q;           // [pages, page_size, KVH, hd * KB / 8]
    half* k_s;              // [pages, page_size, KVH, hd/32]
    uint8_t* v_q;
    half* v_s;
    const int32_t* cache_seqlens;   // [batch]  tokens already in the cache
    const int32_t* block_table;     // [batch, pages_per_seq]
    half* out;              // [batch, q_len, H, hd]
    half* out_xp;           // optional: the consumer matrix's (o_proj) activation buffer, core-matrix layout, permuted rows
    const uint16_t* out_invperm;
    int q_len, H, KVH, hd, page_size, pages_per_seq, max_ctx;
    float scale_log2;       // softmax_scale * log2(e)
    // optional fused RoPE: q and k_new arrive UN-rotated (straight from the Q|K|V projection) and are rotated as they are read,
    // with the fp16 op order of rope_kernel / cuda/rope.cu:52-67,111-122; position of row i = cache_seqlens[b] + i
    const half* rope_sin;   // [max_pos, sincos_size] or NULL
    const half* rope_cos;
    int rope_neox, sincos_size;
    int out_plain;          // out_xp is a plain fp16 row (single-row GEMV consumer) instead of the core-matrix operand layout
    int32_t* err;           // sticky device flag: bit 0 = a sequence ran past its page table (nothing appended, no output)
    // split-KV (long contexts, q_len == 1): grid.z CTAs share one (head, sequence); each attends a contiguous chunk of positions
    // and leaves (max, sum, unnormalised rotated output) in `ws`; the last to arrive (counter) merges.  Chunks are at least
    // AQ_SPLIT_MIN positions, so short contexts use one CTA and never touch the workspace.
    int sc_len;             // floats of the score buffer
    int stage;              // cached positions per CTA copied to shared memory before the dependency wait (the bytes of AQ_STAGE Q4 rows; half with the ring)
    int ring_slots;         // long contexts: cached rows beyond the staged window stream through a ring of sub-chunks (aq_sub) (0: loads from global)
    int batch;              // grid: one CTA per (head, sequence, split), flattened on x, padded to one CTA per SM with slot holders
    int busy_ctas;          //   = H * batch * nsplit
    unsigned int* slot_cnt; // CTAs of this launch that are done (self-resetting), see gemv_i8.cu
    int nsplit;
    float* ws;              // [batch][H][nsplit][hd + 2]
    unsigned int* cnt;      // [batch][H]
    unsigned long long* dbg;   // optional globaltimer stamps of CTA (dbg_cta, 0, 0) (exl2b_debug_set): 0 start, 1 cache rows requested,
    int dbg_cta;               //   2 dependency wait over, 3 new rows quantised / query rotated, 4 scores + max, 5 P V done; 6 / 7 grid span
};
__device__ __forceinline__ unsigned long long aq_gtimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
#define AQ_STAMP(i) do { if (P.dbg) { if (blockIdx.x == P.dbg_cta && threadIdx.x == 0) P.dbg[i] = aq_gtimer(); \
                                      if ((i) == 0 && threadIdx.x == 0) atomicMin(P.dbg + 6, aq_gtimer()); } } while (0)
constexpr int AQ_SPLIT_MIN = 512;
// every exit of a working CTA: count it (slot holders of the launch leave when all working CTAs have)
#define AQ_EXIT do { if (threadIdx.x == 0 && atomicAdd(P.slot_cnt, 1u) == gridDim.x - 1u) *reinterpret_cast<volatile unsigned int*>(P.slot_cnt) = 0u; return; } while (0)
constexpr int AQ_SUB = 128;            // positions per sub-chunk of the streaming ring (long contexts)
constexpr int AQ_RING = 4;             // sub-chunks in flight
constexpr int AQ_STAGE = 512;          // cached positions per CTA staged in shared memory before the dependency wait (Q4; the
                                       // other formats stage the same number of BYTES, host side)

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
template <int BYTES>
__device__ __forceinline__ void cp_async_small(uint32_t dst, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(dst), "l"(src), "n"(BYTES) : "memory");
}

// one half2 (elements un*64 + 2*lane, +1) of a head row, rotated if RoPE is fused.  Warp-uniform call.
template <int HD>
__device__ __forceinline__ half2 load_roped(const half* __restrict__ row, int un, int lane, const AttnQ4Params& P, int pos) {
    const half2 v = reinterpret_cast<const half2*>(row + un * 64)[lane];
    if (!P.rope_sin) return v;
    const half* sr = P.rope_sin + (size_t)pos * P.sincos_size;
    const half* cr = P.rope_cos + (size_t)pos * P.sincos_size;
    if (P.rope_neox) {
        half2 o;
        int col;
        bool first;
        if constexpr (HD == 128) {            // partner element j + 64 lives in the other 64-value unit, same lane
            o = reinterpret_cast<const half2*>(row + (un ^ 1) * 64)[lane];
            col = 2 * lane;
            first = (un == 0);
        } else {                              // HD == 64: partner j + 32 is lane ^ 16
            o = __shfl_xor_sync(0xffffffffu, v, 16);
            col = 2 * (lane & 15);
            first = lane < 16;
        }
        const half2 c2 = *reinterpret_cast<const half2*>(cr + col);
        const half2 s2 = *reinterpret_cast<const half2*>(sr + col);
        if (first) return __hfma2(v, c2, __hmul2(o, __hneg2(s2)));      // l' = l c + half(r * -s)
        return __hfma2(v, c2, __hmul2(o, s2));                            // r' = r c + half(l * s)
    }
    const int col = un * 64 + 2 * lane;
    const half2 c01 = *reinterpret_cast<const half2*>(cr + col);
    half2 s01 = *reinterpret_cast<const half2*>(sr + col);
    uint32_t sb = *reinterpret_cast<uint32_t*>(&s01) ^ (1u << 15);        // (-sin[i], +sin[i+1])
    s01 = *reinterpret_cast<half2*>(&sb);
    return __hfma2(__lowhigh2highlow(v), s01, __hmul2(v, c01));
}

// fp32 Hadamard-32 across the warp on both halves of a float2 (same butterfly as cache_q.cuh, exact sign handling)
__device__ __forceinline__ float2 hadamard32_f(float2 w, int lane) {
#pragma unroll
    for (int i = 1; i < 32; i <<= 1) {
        const float px = __shfl_xor_sync(0xffffffffu, w.x, i), py = __shfl_xor_sync(0xffffffffu, w.y, i);
        const float sg = (lane & i) ? -1.f : 1.f;
        w.x = fmaf(sg, w.x, px);
        w.y = fmaf(sg, w.y, py);
    }
    return w;
}

__device__ __forceinline__ half2 hadamard32_h(half2 w2, int lane) {      // bit-identical to kvcache.cu hadamard32
#pragma unroll
    for (int i = 1; i < 32; i <<= 1) {
        const half2 pw2 = __shfl_xor_sync(0xffffffffu, w2, i);
        uint32_t* w2i = reinterpret_cast<uint32_t*>(&w2);
        const int32_t sfm = -static_cast<int32_t>(lane & i) >> 31;
        *w2i ^= (sfm & 0x80008000);
        w2 = __hadd2(w2, pw2);
    }
    return w2;
}

__device__ __forceinline__ int aq_dp4a_us(uint32_t a, uint32_t b, int c) {      // a: 4 unsigned bytes, b: 4 signed bytes
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
__device__ __forceinline__ int aq_dp4a_uu(uint32_t a, uint32_t b, int c) {
    int d;
    asm("dp4a.u32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

// (nibble - 8) as fp32 without I2F: 0x4B000000 | n is the float 2^23 + n
__device__ __forceinline__ float nib_f(uint32_t n) { return __uint_as_float(0x4B000000u | n) - 8388616.0f; }
// (byte - 128) as fp32, same trick
__device__ __forceinline__ float byte_f(uint32_t n) { return __uint_as_float(0x4B000000u | n) - 8388736.0f; }

template <int KB, int VB>
constexpr int aq_sub() { return AQ_SUB * 4 / (KB > VB ? KB : VB); }      // ring sub-chunk positions: the Q4 sub-chunk's bytes

template <int HD, int KB, int VB>
__global__ void __launch_bounds__(AQ_THREADS, 2) attn_q4_kernel(const __grid_constant__ AttnQ4Params P) {
    static_assert((KB == 4 || KB == 8) && (VB == 4 || VB == 8), "element widths are 4 or 8 bits");
    constexpr int ROWBK = HD * KB / 8;      // packed bytes per (position, kv head): keys
    constexpr int ROWBV = HD * VB / 8;      //   values
    constexpr int ROWB = ROWBK > ROWBV ? ROWBK : ROWBV;     // one ring slot position (keys, then values)
    constexpr int SUB = aq_sub<KB, VB>();
    constexpr int NSC = HD / 32;            // scales per (position, kv head)
    constexpr int VEC = HD / 32;            // values per lane in the dims-on-lanes phase
    constexpr int UNITS = HD / 64;
    extern __shared__ __align__(16) uint8_t smem[];
    const int h = (int)blockIdx.x % P.H, b = ((int)blockIdx.x / P.H) % P.batch, z = (int)blockIdx.x / (P.H * P.batch);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int group = P.H / P.KVH, kvh = h / group;
    __shared__ int s_last;

    constexpr int QPAD = 36;               // floats per 32-value block of the rotated query (bank-staggered: 4 blocks, 4 threads per row)
    constexpr int QIB = 80;                // bytes per 32-value block of the integer query operands (64 used; bank-staggered like QPAD)
    float* qrot = reinterpret_cast<float*>(smem);                          // [NSC][QPAD]
    uint8_t* qi = reinterpret_cast<uint8_t*>(qrot + NSC * QPAD);           // [NSC][QIB]  16-bit query as dp4a byte operands (below)
    int* qsum = reinterpret_cast<int*>(qi + NSC * QIB);                    // [NSC]  sum of a block's 16-bit values
    float* qscl = reinterpret_cast<float*>(qsum + NSC);                    // [NSC]  its power-of-two scale
    float* red = qscl + NSC;                                               // [AQ_WARPS][HD]
    float* wred = red + AQ_WARPS * HD;                                     // [2 * AQ_WARPS]
    uint8_t* new_q = reinterpret_cast<uint8_t*>(wred + 2 * AQ_WARPS);      // [AQ_MAX_QLEN][ROWBK], then [AQ_MAX_QLEN][ROWBV]
    half* new_s = reinterpret_cast<half*>(new_q + AQ_MAX_QLEN * (ROWBK + ROWBV)); // [2][AQ_MAX_QLEN][NSC]
    float* new_y = reinterpret_cast<float*>(new_s + 2 * AQ_MAX_QLEN * NSC);// [2][AQ_MAX_QLEN][HD] rotated, unquantised new rows
    int* pages_s = reinterpret_cast<int*>(new_y + 2 * AQ_MAX_QLEN * HD);   // [pages_per_seq]
    float* sc = reinterpret_cast<float*>(pages_s + ((P.pages_per_seq + 3) & ~3));   // [sc_len]
    uint8_t* kst = reinterpret_cast<uint8_t*>(sc + ((P.sc_len + 3) & ~3));            // [stage][ROWBK]  staged cached K rows
    uint8_t* vst = kst + P.stage * ROWBK;                                            // [stage][ROWBV]
    half* ksst = reinterpret_cast<half*>(vst + P.stage * ROWBV);                     // [stage][NSC]
    half* vsst = ksst + P.stage * NSC;
    uint8_t* rq = reinterpret_cast<uint8_t*>(vsst + P.stage * NSC);                  // [AQ_RING][SUB][ROWB]  streaming ring (K, then V)
    half* rs = reinterpret_cast<half*>(rq + AQ_RING * SUB * ROWB);                   // [AQ_RING][SUB][NSC]

    AQ_STAMP(0);
    griddep_launch_dependents();
    if ((int)blockIdx.x >= P.busy_ctas) {          // slot holder (gemv_i8.cu): keeps this SM's slot until the working CTAs are done
        if (threadIdx.x == 0) {
            while (*reinterpret_cast<volatile unsigned int*>(P.slot_cnt) < (unsigned)P.busy_ctas) __nanosleep(200);
            if (atomicAdd(P.slot_cnt, 1u) == gridDim.x - 1u) *reinterpret_cast<volatile unsigned int*>(P.slot_cnt) = 0u;
        }
        return;
    }
    // ---- 0. before the dependency wait: everything that only touches state written by EARLIER steps / layers -- the
    //      sequence length, the page table and the cached rows (this layer's cache was last written one decode step ago; the
    //      kernel in front of us in the stream, the Q|K|V projection, writes none of it).  The first cached K row of every
    //      thread and the first 16 cached V rows of every warp are already in registers when q / k_new / v_new arrive.
    const int seqlen = P.cache_seqlens[b];
    if (seqlen < 0 || seqlen + P.q_len > P.max_ctx) {      // the page table / score buffer end here: refuse instead of corrupting
        if (tid == 0 && P.err) atomicOr(P.err, 1);
        AQ_EXIT;
    }
    const int32_t* btg = P.block_table + (size_t)b * P.pages_per_seq;
    // this CTA's share of the positions (the whole context unless split-KV is active and the context is long)
    int ns_act = 1, p_lo = 0, p_hi = seqlen + P.q_len;
    if (P.nsplit > 1) {
        const int n_all = seqlen + 1;
        ns_act = min(P.nsplit, max(1, (n_all + AQ_SPLIT_MIN - 1) / AQ_SPLIT_MIN));
        if (z >= ns_act) AQ_EXIT;
        const int chunk = (n_all + ns_act - 1) / ns_act;
        p_lo = z * chunk;
        p_hi = min(n_all, p_lo + chunk);
    }
    const int c_hi = min(p_hi, seqlen);          // cached rows of this CTA: [p_lo, c_hi)
    // The first P.stage cached positions of this CTA are copied to shared memory with cp.async (no registers held across the
    // wait): K / V elements [pos][ROWBK] / [pos][ROWBV] and their fp16 scales [pos][NSC].
    constexpr int TPR = NSC, RPP = AQ_THREADS / TPR;      // scores: NSC threads per position (one 32-value block + scale each)
    const int kblk = tid & (TPR - 1), krow = tid / TPR;
    const int n_st = max(0, min(c_hi - p_lo, P.stage));
    {
        if constexpr (ROWBK == ROWBV) {
            constexpr int CH = ROWB / 16;
            for (int idx = tid; idx < n_st * CH; idx += AQ_THREADS) {
                const int pos = idx / CH, ch = idx - pos * CH, pp = p_lo + pos;
                const int page = btg[pp / P.page_size];
                const size_t row = ((size_t)page * P.page_size + pp % P.page_size) * P.KVH + kvh;
                cp_async16(smem_addr(kst + pos * ROWB + ch * 16), P.k_q + row * ROWB + ch * 16);
                cp_async16(smem_addr(vst + pos * ROWB + ch * 16), P.v_q + row * ROWB + ch * 16);
            }
        } else {
            auto stage_rows = [&](uint8_t* dst, const uint8_t* src, auto rowb) {
                constexpr int RB = decltype(rowb)::value, CH = RB / 16;
                for (int idx = tid; idx < n_st * CH; idx += AQ_THREADS) {
                    const int pos = idx / CH, ch = idx - pos * CH, pp = p_lo + pos;
                    const int page = btg[pp / P.page_size];
                    const size_t row = ((size_t)page * P.page_size + pp % P.page_size) * P.KVH + kvh;
                    cp_async16(smem_addr(dst + pos * RB + ch * 16), src + row * RB + ch * 16);
                }
            };
            stage_rows(kst, P.k_q, std::integral_constant<int, ROWBK>{});
            stage_rows(vst, P.v_q, std::integral_constant<int, ROWBV>{});
        }
        for (int pos = tid; pos < n_st; pos += AQ_THREADS) {
            const int pp = p_lo + pos;
            const int page = btg[pp / P.page_size];
            const size_t row = ((size_t)page * P.page_size + pp % P.page_size) * P.KVH + kvh;
            cp_async_small<NSC * 2>(smem_addr(ksst + pos * NSC), P.k_s + row * NSC);
            cp_async_small<NSC * 2>(smem_addr(vsst + pos * NSC), P.v_s + row * NSC);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    for (int i = tid; i < P.pages_per_seq; i += AQ_THREADS) pages_s[i] = btg[i];
    const int* bt = pages_s;
    // sub-chunk t of the cached rows beyond the staged window -> ring slot t % AQ_RING (one cp.async group per call, possibly empty);
    // rows of RB bytes (keys, then values) at a pitch of ROWB
    auto ring_issue = [&](int t, const uint8_t* gq, const half* gs, auto rowb) {
        constexpr int RB = decltype(rowb)::value;
        const int base = p_lo + n_st + t * SUB, cnt = min(SUB, c_hi - base), slot = t & (AQ_RING - 1);
        if (cnt > 0) {
            constexpr int CH = RB / 16;
            for (int idx = tid; idx < cnt * CH; idx += AQ_THREADS) {
                const int pos = idx / CH, ch = idx - pos * CH, pp = base + pos;
                const int page = bt[pp / P.page_size];
                const size_t row = ((size_t)page * P.page_size + pp % P.page_size) * P.KVH + kvh;
                cp_async16(smem_addr(rq + (slot * SUB + pos) * ROWB + ch * 16), gq + row * RB + ch * 16);
            }
            for (int pos = tid; pos < cnt; pos += AQ_THREADS) {
                const int pp = base + pos;
                const int page = bt[pp / P.page_size];
                const size_t row = ((size_t)page * P.page_size + pp % P.page_size) * P.KVH + kvh;
                cp_async_small<NSC * 2>(smem_addr(rs + (slot * SUB + pos) * NSC), gs + row * NSC);
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    const int ntail = (P.ring_slots && c_hi > p_lo + n_st) ? (c_hi - (p_lo + n_st) + SUB - 1) / SUB : 0;
    AQ_STAMP(1);
    griddep_wait();
    AQ_STAMP(2);

    // ---- 1. quantise the new rows (fp16_to_q_kv arithmetic) on the first warps, keep them in shared memory; at the same
    //      time the LAST warps rotate the first query: qrot = H q * (softmax_scale * log2 e / 32)
    auto rotate_q = [&](int i, int un) {
        const half2 qh = load_roped<HD>(P.q + (((size_t)b * P.q_len + i) * P.H + h) * HD, un, lane, P, seqlen + i);
        float2 w = hadamard32_f(__half22float2(qh), lane);
        const float f = P.scale_log2 * (1.0f / 32.0f);
        const int e = un * 64 + 2 * lane;
        w.x *= f;
        w.y *= f;
        qrot[(e >> 5) * QPAD + (e & 31)] = w.x;
        qrot[(e >> 5) * QPAD + (e & 31) + 1] = w.y;
        // The cached rows are scored on the integer dot-product instruction (like the batch-1 GEMV): the block's 32 values as 16-bit
        // integers with a power-of-two scale (error <= 2^-15 of the block maximum), split into a signed high and an unsigned low
        // byte plane, bytes ordered as the masked nibble words of a cached row present them: word j of a block holds values 8j..8j+7,
        // (x & 0x0f0f0f0f) = values 8j + {0,2,4,6}, (x & 0xf0f0f0f0) = 16 * values 8j + {1,3,5,7}.
        float amax = fmaxf(fabsf(w.x), fabsf(w.y));
#pragma unroll
        for (int o = 1; o < 16; o <<= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));      // 16 lanes = one block
        const uint32_t ef = (__float_as_uint(amax * 1.000030518f) >> 23) & 0xffu;
        const float inv = amax > 0.f ? __uint_as_float((268u - ef) << 23) : 0.f;
        const uint32_t q0 = __float_as_uint(fmaf(w.x, inv, 12582912.f)), q1 = __float_as_uint(fmaf(w.y, inv, 12582912.f));
        int sum = (int)(q0 + q1 - 2u * 0x4B400000u);
#pragma unroll
        for (int o = 1; o < 16; o <<= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        const int blk = e >> 5, l16 = lane & 15;
        if constexpr (KB == 4) {
            const int j = l16 >> 2, m = l16 & 3;
            uint8_t* qb = qi + blk * QIB + j * 16 + m;          // word order per j: even-high, even-low, odd-high, odd-low
            qb[0] = (uint8_t)(q0 >> 8);
            qb[4] = (uint8_t)q0;
            qb[8] = (uint8_t)(q1 >> 8);
            qb[12] = (uint8_t)q1;
        } else {
            // 8-bit keys: word w of a block holds values 4w..4w+3 in byte order; per pair of words j = w / 2 the 16 bytes are
            // high(w = 2j), low(2j), high(2j + 1), low(2j + 1).  This lane's values 2 l16, 2 l16 + 1 sit in word l16 / 2.
            const int w8 = l16 >> 1;
            uint8_t* qb = qi + blk * QIB + (w8 >> 1) * 16 + (w8 & 1) * 8 + (l16 & 1) * 2;
            qb[0] = (uint8_t)(q0 >> 8);
            qb[1] = (uint8_t)(q1 >> 8);
            qb[4] = (uint8_t)q0;
            qb[5] = (uint8_t)q1;
        }
        if (l16 == 0) {
            qsum[blk] = sum;
            qscl[blk] = amax > 0.f ? __uint_as_float((ef - 14u) << 23) : 0.f;
        }
    };
    if (warp >= AQ_WARPS - UNITS) rotate_q(0, warp - (AQ_WARPS - UNITS));
    const int n_jobs = 2 * P.q_len * UNITS;
    for (int job = (warp >= AQ_WARPS - UNITS && n_jobs <= AQ_WARPS - UNITS) ? n_jobs : warp; job < n_jobs; job += AQ_WARPS) {
        const int kv = job / (P.q_len * UNITS), r = job - kv * P.q_len * UNITS;
        const int i = r / UNITS, un = r - i * UNITS;
        const half* src = (kv ? P.v_new : P.k_new) + (((size_t)b * P.q_len + i) * P.KVH + kvh) * HD;
        half2 w2 = kv ? reinterpret_cast<const half2*>(src + un * 64)[lane] : load_roped<HD>(src, un, lane, P, seqlen + i);
        {
            const float2 y = hadamard32_f(__half22float2(w2), lane);
            new_y[(kv * AQ_MAX_QLEN + i) * HD + un * 64 + 2 * lane] = y.x;
            new_y[(kv * AQ_MAX_QLEN + i) * HD + un * 64 + 2 * lane + 1] = y.y;
        }
        w2 = hadamard32_h(w2, lane);
        half2 absmax2 = __habs2(w2);
        half absmax = __hmax(__low2half(absmax2), __high2half(absmax2));
        absmax = __hmax(absmax, __shfl_xor_sync(0xffffffffu, absmax, 8));
        absmax = __hmax(absmax, __shfl_xor_sync(0xffffffffu, absmax, 4));
        absmax = __hmax(absmax, __shfl_xor_sync(0xffffffffu, absmax, 2));
        absmax = __hmax(absmax, __shfl_xor_sync(0xffffffffu, absmax, 1));
        uint8_t* nq = new_q + (kv ? AQ_MAX_QLEN * ROWBK + i * ROWBV : i * ROWBK);
        if ((kv ? VB : KB) == 4) {
            const half2 c_8 = __half2half2(__float2half_rn(8));
            w2 = __h2div(w2, __half2half2(absmax));
            w2 = __hfma2(w2, c_8, c_8);
            const int q0 = min(max(__half2int_rn(__low2half(w2)), 0), 15);
            const int q1 = min(max(__half2int_rn(__high2half(w2)), 0), 15);
            nq[un * 32 + lane] = (uint8_t)(q0 | (q1 << 4));
            if ((lane & 15) == 0) new_s[(kv * AQ_MAX_QLEN + i) * NSC + un * 2 + (lane >> 4)] = __hmul(absmax, __float2half_rn(1.0f / 8.0f));
        } else {                                  // 8 bits (kvcache.cu pack_unit_q8)
            const half2 c_128 = __half2half2(__float2half_rn(128));
            w2 = __h2div(w2, __half2half2(absmax));
            w2 = __hfma2(w2, c_128, c_128);
            const int q0 = min(max(__half2int_rn(__low2half(w2)), 0), 255);
            const int q1 = min(max(__half2int_rn(__high2half(w2)), 0), 255);
            reinterpret_cast<uint16_t*>(nq + un * 64)[lane] = (uint16_t)(q0 | (q1 << 8));
            if ((lane & 15) == 0) new_s[(kv * AQ_MAX_QLEN + i) * NSC + un * 2 + (lane >> 4)] = __hmul(absmax, __float2half_rn(1.0f / 128.0f));
        }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    AQ_STAMP(3);
    AQ_STAMP(8);

    // score of one 32-value block of a cached row (one fp16 scale) against its block of the rotated query, all in integers (dp4a),
    // one fp32 multiply at the end.  4 bits: sum_d (nib_d - 8) q_d = sum nib q - 8 sum q, dp4a on the masked words.
    // 8 bits: sum_d (b_d - 128) q_d = sum b q - 128 sum q, dp4a on the stored words as they are.  The offset is removed with the
    // block's query sum (one multiply-add per block, shared with the 4-bit path) rather than by flipping every byte's top bit and
    // using signed dp4a (one extra logic op per word, 8 per block).
    constexpr int KW = KB / 4;               // uint4 words per 32-value key block
    constexpr uint32_t KFILL = KB == 4 ? 0x88888888u : 0x80808080u;      // a zero block (never scored: keeps registers defined)
    auto score_blk = [&](const uint4* kq, uint32_t ks) {
        const uint8_t* qb = qi + kblk * QIB;
        int v;
        if constexpr (KB == 4) {
            const uint32_t ww[4] = {kq[0].x, kq[0].y, kq[0].z, kq[0].w};
            int a0 = 0, a1 = 0, a2 = 0, a3 = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint4 qo = *reinterpret_cast<const uint4*>(qb + j * 16);
                const uint32_t lo = ww[j] & 0x0f0f0f0fu, hi = ww[j] & 0xf0f0f0f0u;
                a0 = aq_dp4a_us(lo, qo.x, a0);          // unsigned nibbles x signed high bytes
                a1 = aq_dp4a_uu(lo, qo.y, a1);          // unsigned x unsigned low bytes
                a2 = aq_dp4a_us(hi, qo.z, a2);
                a3 = aq_dp4a_uu(hi, qo.w, a3);
            }
            v = ((a0 << 8) + a1) + (((a2 << 8) + a3) >> 4) - 8 * qsum[kblk];
        } else {
            const uint32_t ww[8] = {kq[0].x, kq[0].y, kq[0].z, kq[0].w, kq[1].x, kq[1].y, kq[1].z, kq[1].w};
            int a0 = 0, a1 = 0, a2 = 0, a3 = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint4 qo = *reinterpret_cast<const uint4*>(qb + j * 16);
                a0 = aq_dp4a_us(ww[2 * j], qo.x, a0);          // unsigned bytes x signed high bytes
                a1 = aq_dp4a_uu(ww[2 * j], qo.y, a1);          // unsigned x unsigned low bytes
                a2 = aq_dp4a_us(ww[2 * j + 1], qo.z, a2);
                a3 = aq_dp4a_uu(ww[2 * j + 1], qo.w, a3);
            }
            v = ((a0 + a2) << 8) + (a1 + a3) - 128 * qsum[kblk];
        }
        return __half2float(__ushort_as_half((unsigned short)ks)) * qscl[kblk] * (float)v;
    };

    for (int i = 0; i < P.q_len; ++i) {
        const int n_ctx = (P.nsplit > 1) ? p_hi : seqlen + i + 1;          // end of the positions this CTA attends for query i
        if (i > 0) {                         // (the first query was rotated above, next to the quantisation)
            if (warp < UNITS) rotate_q(i, warp);
            __syncthreads();
        }

        // ---- 2. scores: NSC threads per position, each its 32-value block of the (rotated) row against qrot ----
        float lmax = -INFINITY;
        auto score_pos = [&](int p, const uint4* kq, uint32_t ks) {      // warp-uniform call (the NSC partial sums meet by shuffle)
            float s = 0.f;
            if (p < n_ctx) {
                if (p >= seqlen) {               // a row appended by this step: fp16 values, rotated in fp32
                    const float4* y4 = reinterpret_cast<const float4*>(new_y + (p - seqlen) * HD + kblk * 32);
                    const float4* q4 = reinterpret_cast<const float4*>(qrot + kblk * QPAD);
                    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const float4 a = q4[j], c = y4[j];
                        s0 = fmaf(a.x, c.x, s0);
                        s1 = fmaf(a.y, c.y, s1);
                        s2 = fmaf(a.z, c.z, s2);
                        s3 = fmaf(a.w, c.w, s3);
                    }
                    s = (s0 + s1) + (s2 + s3);
                } else {
                    s = score_blk(kq, ks);
                }
            }
#pragma unroll
            for (int o = 1; o < TPR; o <<= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (p < n_ctx) {
                if (kblk == 0) sc[p - p_lo] = s;
                lmax = fmaxf(lmax, s);
            }
        };
        {
            const int st_end = p_lo + n_st;                      // positions below are in shared memory
            int pb = p_lo;
            for (; pb < n_ctx && pb < st_end; pb += RPP) {
                const int pp = pb + krow;
                uint4 kq[KW];
#pragma unroll
                for (int u = 0; u < KW; ++u) kq[u] = make_uint4(KFILL, KFILL, KFILL, KFILL);
                uint32_t ks = 0u;
                if (pp < st_end) {
#pragma unroll
                    for (int u = 0; u < KW; ++u) kq[u] = reinterpret_cast<const uint4*>(kst + (pp - p_lo) * ROWBK)[kblk * KW + u];
                    ks = *reinterpret_cast<const unsigned short*>(ksst + (pp - p_lo) * NSC + kblk);
                } else if (pp < min(n_ctx, seqlen)) {
                    const int page = bt[pp / P.page_size];
                    const size_t row = ((size_t)page * P.page_size + pp % P.page_size) * P.KVH + kvh;
#pragma unroll
                    for (int u = 0; u < KW; ++u) kq[u] = __ldg(reinterpret_cast<const uint4*>(P.k_q + row * ROWBK) + kblk * KW + u);
                    ks = __ldg(reinterpret_cast<const unsigned short*>(P.k_s + row * NSC) + kblk);
                }
                score_pos(pp, kq, ks);
            }
            if (ntail > 0) {
                // long context: the remaining cached K rows stream through the ring, AQ_RING sub-chunks in flight
                __syncthreads();                                  // (every thread is done with the ring's previous contents)
                for (int t = 0; t < AQ_RING; ++t) ring_issue(t, P.k_q, P.k_s, std::integral_constant<int, ROWBK>{});
                for (int t = 0; t < ntail; ++t) {
                    asm volatile("cp.async.wait_group %0;" ::"n"(AQ_RING - 1) : "memory");
                    __syncthreads();
                    const int base = p_lo + n_st + t * SUB, slot = t & (AQ_RING - 1);
#pragma unroll 1
                    for (int r0 = 0; r0 < SUB; r0 += RPP) {
                        if (base + r0 >= n_ctx) break;
                        const int rr = r0 + krow, pp = base + rr;
                        // an 8-bit sub-chunk can hold fewer positions than one pass scores (hd 64: 64 < RPP = 128): rows past
                        // the sub-chunk belong to the next one and are neither read nor scored here
                        const bool in_sub = SUB >= RPP || rr < SUB;
                        uint4 kq[KW];
#pragma unroll
                        for (int u = 0; u < KW; ++u) kq[u] = make_uint4(KFILL, KFILL, KFILL, KFILL);
                        uint32_t ks = 0u;
                        if (in_sub && pp < c_hi) {
#pragma unroll
                            for (int u = 0; u < KW; ++u) kq[u] = reinterpret_cast<const uint4*>(rq + (slot * SUB + rr) * ROWB)[kblk * KW + u];
                            ks = *reinterpret_cast<const unsigned short*>(rs + (slot * SUB + rr) * NSC + kblk);
                        }
                        score_pos(in_sub ? pp : INT_MAX, kq, ks);
                    }
                    __syncthreads();
                    ring_issue(t + AQ_RING, P.k_q, P.k_s, std::integral_constant<int, ROWBK>{});
                }
                pb = p_lo + n_st + ntail * SUB;
            }
            constexpr int TU = 2 / KW;                           // rows per thread in flight: 32 bytes of keys in every format
            for (; pb < n_ctx; pb += TU * RPP) {                 // rows appended by this step; without the ring: everything beyond the window
                uint4 kq[TU][KW];
                uint32_t ks[TU];
#pragma unroll
                for (int u = 0; u < TU; ++u) {
                    const int pp = pb + u * RPP + krow;
#pragma unroll
                    for (int w = 0; w < KW; ++w) kq[u][w] = make_uint4(KFILL, KFILL, KFILL, KFILL);
                    ks[u] = 0u;
                    if (pp < min(n_ctx, seqlen)) {
                        const int page = bt[pp / P.page_size];
                        const size_t row = ((size_t)page * P.page_size + pp % P.page_size) * P.KVH + kvh;
#pragma unroll
                        for (int w = 0; w < KW; ++w) kq[u][w] = __ldg(reinterpret_cast<const uint4*>(P.k_q + row * ROWBK) + kblk * KW + w);
                        ks[u] = __ldg(reinterpret_cast<const unsigned short*>(P.k_s + row * NSC) + kblk);
                    }
                }
#pragma unroll
                for (int u = 0; u < TU; ++u)
                    if (pb + u * RPP < n_ctx) score_pos(pb + u * RPP + krow, kq[u], ks[u]);
            }
        }
        AQ_STAMP(9);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
        if (lane == 0) wred[warp] = lmax;
        __syncthreads();
        AQ_STAMP(4);
        float mx = wred[0];
#pragma unroll
        for (int w = 1; w < AQ_WARPS; ++w) mx = fmaxf(mx, wred[w]);
        float lsum = 0.f;
        for (int p = p_lo + tid; p < n_ctx; p += AQ_THREADS) {
            const float e = exp2f(sc[p - p_lo] - mx);
            sc[p - p_lo] = e;
            lsum += e;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
        if (lane == 0) wred[AQ_WARPS + warp] = lsum;
        __syncthreads();
        float denom = 0.f;
#pragma unroll
        for (int w = 0; w < AQ_WARPS; ++w) denom += wred[AQ_WARPS + w];

        // ---- 3. P V in the rotated domain: lane = VEC consecutive values, warps stride over positions ----
        float acc[VEC];
#pragma unroll
        for (int j = 0; j < VEC; ++j) acc[j] = 0.f;
        auto pv_fma = [&](uint32_t xs, float pw) {                           // 4-bit values: nibbles | scale << 16
            const float pe = pw * __half2float(__ushort_as_half((unsigned short)(xs >> 16)));
            if constexpr (VEC == 4) {
                acc[0] = fmaf(pe, nib_f(xs & 15u), acc[0]);
                acc[1] = fmaf(pe, nib_f((xs >> 4) & 15u), acc[1]);
                acc[2] = fmaf(pe, nib_f((xs >> 8) & 15u), acc[2]);
                acc[3] = fmaf(pe, nib_f((xs >> 12) & 15u), acc[3]);
            } else {
                acc[0] = fmaf(pe, nib_f(xs & 15u), acc[0]);
                acc[1] = fmaf(pe, nib_f((xs >> 4) & 15u), acc[1]);
            }
        };
        auto pv_fma8 = [&](uint32_t xd, uint32_t xs, float pw) {             // 8-bit values: VEC bytes in xd, scale in xs
            const float pe = pw * __half2float(__ushort_as_half((unsigned short)xs));
#pragma unroll
            for (int j = 0; j < VEC; ++j) acc[j] = fmaf(pe, byte_f((xd >> (8 * j)) & 0xffu), acc[j]);
        };
        auto v8_smem = [&](const uint8_t* rowp) -> uint32_t {               // this lane's VEC bytes of an 8-bit row
            if constexpr (VEC == 4) return *reinterpret_cast<const uint32_t*>(rowp + lane * 4);
            else return *reinterpret_cast<const uint16_t*>(rowp + lane * 2);
        };
        {
            const int st_end = p_lo + n_st;                      // staged rows: shared memory
#pragma unroll 4
            for (int p = p_lo + warp; p < st_end; p += AQ_WARPS) {
                const int r = p - p_lo;
                if constexpr (VB == 4) {
                    uint32_t x;
                    if constexpr (VEC == 4) x = *reinterpret_cast<const uint16_t*>(vst + r * ROWBV + lane * 2);
                    else x = (uint32_t)vst[r * ROWBV + lane] | 0x8800u;
                    x |= (uint32_t)(*reinterpret_cast<const uint16_t*>(vsst + r * NSC + ((lane * VEC) >> 5))) << 16;
                    pv_fma(x, sc[r]);
                } else {
                    pv_fma8(v8_smem(vst + r * ROWBV), *reinterpret_cast<const uint16_t*>(vsst + r * NSC + ((lane * VEC) >> 5)), sc[r]);
                }
            }
        }
        if (ntail > 0) {
            // long context: the remaining cached V rows through the same ring
            __syncthreads();
            for (int t = 0; t < AQ_RING; ++t) ring_issue(t, P.v_q, P.v_s, std::integral_constant<int, ROWBV>{});
            for (int t = 0; t < ntail; ++t) {
                asm volatile("cp.async.wait_group %0;" ::"n"(AQ_RING - 1) : "memory");
                __syncthreads();
                const int base = p_lo + n_st + t * SUB, slot = t & (AQ_RING - 1);
#pragma unroll 4
                for (int r = warp; r < SUB; r += AQ_WARPS) {
                    const int pp = base + r;
                    if (pp < c_hi) {
                        const uint16_t xsc = *reinterpret_cast<const uint16_t*>(rs + (slot * SUB + r) * NSC + ((lane * VEC) >> 5));
                        if constexpr (VB == 4) {
                            uint32_t x;
                            if constexpr (VEC == 4) x = *reinterpret_cast<const uint16_t*>(rq + (slot * SUB + r) * ROWB + lane * 2);
                            else x = (uint32_t)rq[(slot * SUB + r) * ROWB + lane] | 0x8800u;
                            x |= (uint32_t)xsc << 16;
                            pv_fma(x, sc[pp - p_lo]);
                        } else {
                            pv_fma8(v8_smem(rq + (slot * SUB + r) * ROWB), xsc, sc[pp - p_lo]);
                        }
                    }
                }
                __syncthreads();
                ring_issue(t + AQ_RING, P.v_q, P.v_s, std::integral_constant<int, ROWBV>{});
            }
        }
        for (int p0 = (ntail > 0 ? c_hi : p_lo + n_st) + warp; p0 < c_hi; p0 += AQ_WARPS * 8) {   // without the ring: 8 rows in flight from global
            uint32_t xs[8], xd[VB == 8 ? 8 : 1];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int p = p0 + u * AQ_WARPS;
                if constexpr (VB == 4) xs[u] = 0x8888u;
                else { xs[u] = 0u; xd[u] = 0x80808080u; }
                if (p < c_hi) {
                    const int page = bt[p / P.page_size];
                    const size_t row = ((size_t)page * P.page_size + p % P.page_size) * P.KVH + kvh;
                    if constexpr (VB == 4) {
                        uint32_t x;
                        if constexpr (VEC == 4) x = __ldg(reinterpret_cast<const uint16_t*>(P.v_q + row * ROWBV + lane * 2));
                        else x = (uint32_t)__ldg(P.v_q + row * ROWBV + lane) | 0x8800u;
                        xs[u] = x | ((uint32_t)__ldg(reinterpret_cast<const uint16_t*>(P.v_s + row * NSC + ((lane * VEC) >> 5))) << 16);
                    } else {
                        const uint32_t xsc = __ldg(reinterpret_cast<const uint16_t*>(P.v_s + row * NSC + ((lane * VEC) >> 5)));
                        if constexpr (VEC == 4) xd[u] = __ldg(reinterpret_cast<const uint32_t*>(P.v_q + row * ROWBV) + lane);
                        else xd[u] = __ldg(reinterpret_cast<const uint16_t*>(P.v_q + row * ROWBV) + lane);
                        xs[u] = xsc;
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int p = p0 + u * AQ_WARPS;
                if (p < c_hi) {
                    if constexpr (VB == 4) pv_fma(xs[u], sc[p - p_lo]);
                    else pv_fma8(xd[u], xs[u], sc[p - p_lo]);
                }
            }
        }
        if (warp == 0) {                                                      // rows appended by this step (<= 8)
            for (int p = max(seqlen, p_lo); p < n_ctx; ++p) {
                const float pe = sc[p - p_lo];
                const float* y = new_y + (AQ_MAX_QLEN + p - seqlen) * HD + lane * VEC;
#pragma unroll
                for (int j = 0; j < VEC; ++j) acc[j] = fmaf(pe, y[j], acc[j]);
            }
        }
#pragma unroll
        for (int j = 0; j < VEC; ++j) red[warp * HD + lane * VEC + j] = acc[j];
        __syncthreads();
        AQ_STAMP(5);
        // the rows appended by this step go to the cache now, from shared memory, by the last warp (it has no part in the reduction
        // below): nothing on the way to the output waits for these stores
        if (i == P.q_len - 1 && warp == AQ_WARPS - 1 && h % group == 0 && z == 0) {
            if constexpr (ROWBK == ROWBV) {
                for (int idx = lane; idx < 2 * P.q_len * (ROWB / 4); idx += 32) {
                    const int kv = idx / (P.q_len * (ROWB / 4)), r = idx - kv * P.q_len * (ROWB / 4);
                    const int ii = r / (ROWB / 4), wd = r - ii * (ROWB / 4);
                    const int pos = seqlen + ii;
                    const int page = bt[pos / P.page_size];
                    const size_t row = ((size_t)page * P.page_size + pos % P.page_size) * P.KVH + kvh;
                    reinterpret_cast<uint32_t*>((kv ? P.v_q : P.k_q) + row * ROWB)[wd] =
                        reinterpret_cast<const uint32_t*>(new_q + (kv * AQ_MAX_QLEN + ii) * ROWB)[wd];
                }
            } else {
                constexpr int WK = ROWBK / 4, WV = ROWBV / 4;                 // 32-bit words per key / value row
                for (int idx = lane; idx < P.q_len * (WK + WV); idx += 32) {
                    const int kv = idx >= P.q_len * WK, r = kv ? idx - P.q_len * WK : idx;
                    const int ii = kv ? r / WV : r / WK, wd = kv ? r - ii * WV : r - ii * WK;
                    const int pos = seqlen + ii;
                    const int page = bt[pos / P.page_size];
                    const size_t row = ((size_t)page * P.page_size + pos % P.page_size) * P.KVH + kvh;
                    reinterpret_cast<uint32_t*>(kv ? P.v_q + row * ROWBV : P.k_q + row * ROWBK)[wd] =
                        reinterpret_cast<const uint32_t*>(new_q + (kv ? AQ_MAX_QLEN * ROWBK + ii * ROWBV : ii * ROWBK))[wd];
                }
            }
            for (int idx = lane; idx < 2 * P.q_len * NSC; idx += 32) {
                const int kv = idx / (P.q_len * NSC), r = idx - kv * P.q_len * NSC;
                const int ii = r / NSC, sidx = r - ii * NSC;
                const int pos = seqlen + ii;
                const int page = bt[pos / P.page_size];
                const size_t row = ((size_t)page * P.page_size + pos % P.page_size) * P.KVH + kvh;
                (kv ? P.v_s : P.k_s)[row * NSC + sidx] = new_s[(kv * AQ_MAX_QLEN + ii) * NSC + sidx];
            }
        }
        // ---- 5. sum over warps, (merge the splits,) rotate back (x = H y / 32), normalise, store ----
        if (ns_act > 1) {
            // leave (unnormalised rotated output, max, sum) of this chunk; the last CTA of the (head, sequence) merges them all
            float* wsp = P.ws + (((size_t)b * P.H + h) * P.nsplit + z) * (HD + 2);
            if (warp < UNITS) {
                float2 w = make_float2(0.f, 0.f);
#pragma unroll
                for (int ww = 0; ww < AQ_WARPS; ++ww) {
                    w.x += red[ww * HD + warp * 64 + 2 * lane];
                    w.y += red[ww * HD + warp * 64 + 2 * lane + 1];
                }
                __stcg(reinterpret_cast<float2*>(wsp + warp * 64) + lane, w);
            }
            if (tid == 0) { __stcg(wsp + HD, mx); __stcg(wsp + HD + 1, denom); }
            __threadfence();
            __syncthreads();
            if (tid == 0) {
                const unsigned old = atomicAdd(P.cnt + (size_t)b * P.H + h, 1u);
                s_last = (old == (unsigned)ns_act - 1u);
                if (s_last) P.cnt[(size_t)b * P.H + h] = 0u;
                __threadfence();
            }
            __syncthreads();
            if (!s_last) AQ_EXIT;
            if (warp < UNITS) {
                const float* base = P.ws + ((size_t)b * P.H + h) * P.nsplit * (HD + 2);
                float M = -INFINITY;
                for (int sidx = 0; sidx < ns_act; ++sidx) M = fmaxf(M, __ldcg(base + (size_t)sidx * (HD + 2) + HD));
                float2 w = make_float2(0.f, 0.f);
                float L = 0.f;
                for (int sidx = 0; sidx < ns_act; ++sidx) {
                    const float* ps = base + (size_t)sidx * (HD + 2);
                    const float wgt = exp2f(__ldcg(ps + HD) - M);
                    const float2 a = __ldcg(reinterpret_cast<const float2*>(ps + warp * 64) + lane);
                    w.x = fmaf(wgt, a.x, w.x);
                    w.y = fmaf(wgt, a.y, w.y);
                    L = fmaf(wgt, __ldcg(ps + HD + 1), L);
                }
                w = hadamard32_f(w, lane);
                const float f = (1.0f / 32.0f) / L;
                const half2 o2 = __floats2half2_rn(w.x * f, w.y * f);
                reinterpret_cast<half2*>(P.out + (((size_t)b * P.q_len + i) * P.H + h) * HD + warp * 64)[lane] = o2;
                if (P.out_xp) {
                    const int n = h * HD + warp * 64 + 2 * lane, m = b * P.q_len + i;
                    const int k0 = P.out_invperm ? (int)P.out_invperm[n] : n, k1 = P.out_invperm ? (int)P.out_invperm[n + 1] : n + 1;
                    if (P.out_plain) {
                        P.out_xp[k0] = __low2half(o2);
                        P.out_xp[k1] = __high2half(o2);
                    } else {
                        P.out_xp[(size_t)(k0 >> 3) * 64 + m * 8 + (k0 & 7)] = __low2half(o2);
                        P.out_xp[(size_t)(k1 >> 3) * 64 + m * 8 + (k1 & 7)] = __high2half(o2);
                    }
                }
            }
            AQ_EXIT;
        }
        if (warp < UNITS) {
            float2 w = make_float2(0.f, 0.f);
#pragma unroll
            for (int ww = 0; ww < AQ_WARPS; ++ww) {
                w.x += red[ww * HD + warp * 64 + 2 * lane];
                w.y += red[ww * HD + warp * 64 + 2 * lane + 1];
            }
            w = hadamard32_f(w, lane);
            const float f = (1.0f / 32.0f) / denom;
            const half2 o2 = __floats2half2_rn(w.x * f, w.y * f);
            reinterpret_cast<half2*>(P.out + (((size_t)b * P.q_len + i) * P.H + h) * HD + warp * 64)[lane] = o2;
            if (P.out_xp) {
                const int n = h * HD + warp * 64 + 2 * lane, m = b * P.q_len + i;
                const int k0 = P.out_invperm ? (int)P.out_invperm[n] : n, k1 = P.out_invperm ? (int)P.out_invperm[n + 1] : n + 1;
                if (P.out_plain) {
                    P.out_xp[k0] = __low2half(o2);
                    P.out_xp[k1] = __high2half(o2);
                } else {
                    P.out_xp[(size_t)(k0 >> 3) * 64 + m * 8 + (k0 & 7)] = __low2half(o2);
                    P.out_xp[(size_t)(k1 >> 3) * 64 + m * 8 + (k1 & 7)] = __high2half(o2);
                }
            }
        }
        __syncthreads();
    }
    if (P.dbg && threadIdx.x == 0) atomicMax(P.dbg + 7, aq_gtimer());
    AQ_EXIT;
}

}  // namespace exl2b

using namespace exl2b;

static int32_t* g_attn_err[64] = {nullptr};

extern "C" int exl2b_paged_attn_status(int device, int* status) {
    EXL2B_REQUIRE(status && device >= 0 && device < 64, "bad argument");
    *status = 0;
    if (!g_attn_err[device]) return 0;
    EXL2B_CUDA(cudaSetDevice(device));
    EXL2B_CUDA(cudaMemcpy(status, g_attn_err[device], sizeof(int), cudaMemcpyDeviceToHost));
    return 0;
}

extern "C" int exl2b_paged_attn_clear_status(int device) {
    EXL2B_REQUIRE(device >= 0 && device < 64, "bad argument");
    if (!g_attn_err[device]) return 0;
    EXL2B_CUDA(cudaSetDevice(device));
    EXL2B_CUDA(cudaMemset(g_attn_err[device], 0, sizeof(int)));
    return 0;
}

extern "C" int exl2b_paged_attn_decode_q4(const uint16_t* q, const uint16_t* k_new, const uint16_t* v_new, uint8_t* k_cache,
                                          uint16_t* k_scales, uint8_t* v_cache, uint16_t* v_scales, const int32_t* cache_seqlens,
                                          const int32_t* block_table, uint16_t* out, int batch, int q_len, int num_heads,
                                          int num_kv_heads, int head_dim, int page_size, int pages_per_seq, float softmax_scale,
                                          exl2b_qmatrix_t out_consumer, exl2b_stream_t stream) {
    return exl2b_paged_attn_decode_q4_ex(q, k_new, v_new, k_cache, k_scales, v_cache, v_scales, cache_seqlens, block_table, out, batch,
                                         q_len, num_heads, num_kv_heads, head_dim, page_size, pages_per_seq, softmax_scale, out_consumer,
                                         nullptr, nullptr, 0, 0, stream);
}

extern "C" int exl2b_paged_attn_decode_q4_ex(const uint16_t* q, const uint16_t* k_new, const uint16_t* v_new, uint8_t* k_cache,
                                             uint16_t* k_scales, uint8_t* v_cache, uint16_t* v_scales, const int32_t* cache_seqlens,
                                             const int32_t* block_table, uint16_t* out, int batch, int q_len, int num_heads,
                                             int num_kv_heads, int head_dim, int page_size, int pages_per_seq, float softmax_scale,
                                             exl2b_qmatrix_t out_consumer, const uint16_t* rope_sin, const uint16_t* rope_cos,
                                             int rope_style, int sincos_size, exl2b_stream_t stream) {
    return exl2b_paged_attn_decode_q(q, k_new, v_new, k_cache, k_scales, v_cache, v_scales, cache_seqlens, block_table, out, batch, q_len,
                                     num_heads, num_kv_heads, head_dim, page_size, pages_per_seq, softmax_scale, out_consumer, rope_sin,
                                     rope_cos, rope_style, sincos_size, 4, stream);
}

template <int KB, int VB>
static int attn_q_launch(int head_dim, dim3 grid, size_t smem, cudaStream_t stream, const AttnQ4Params& P) {
    if (head_dim == 128)
        EXL2B_CUDA(launch_pdl_f("attn", attn_q4_kernel<128, KB, VB>, grid, dim3(AQ_THREADS), smem, stream, P));
    else
        EXL2B_CUDA(launch_pdl_f("attn", attn_q4_kernel<64, KB, VB>, grid, dim3(AQ_THREADS), smem, stream, P));
    return 0;
}

template <int KB, int VB>
static int attn_q_set_smem() {
    EXL2B_CUDA(cudaFuncSetAttribute(attn_q4_kernel<128, KB, VB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    EXL2B_CUDA(cudaFuncSetAttribute(attn_q4_kernel<64, KB, VB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    return 0;
}

extern "C" int exl2b_paged_attn_decode_q(const uint16_t* q, const uint16_t* k_new, const uint16_t* v_new, uint8_t* k_cache,
                                         uint16_t* k_scales, uint8_t* v_cache, uint16_t* v_scales, const int32_t* cache_seqlens,
                                         const int32_t* block_table, uint16_t* out, int batch, int q_len, int num_heads,
                                         int num_kv_heads, int head_dim, int page_size, int pages_per_seq, float softmax_scale,
                                         exl2b_qmatrix_t out_consumer, const uint16_t* rope_sin, const uint16_t* rope_cos,
                                         int rope_style, int sincos_size, int wbits, exl2b_stream_t stream) {
    EXL2B_REQUIRE(q && k_new && v_new && k_cache && k_scales && v_cache && v_scales && cache_seqlens && block_table && out, "null argument");
    EXL2B_REQUIRE(wbits == 4 || wbits == 6 || wbits == 8, "cache wbits must be 4 (Q4), 6 (Q6) or 8 (Q8); got %d", wbits);
    const int kb = wbits == 4 ? 4 : 8, vb = wbits == 8 ? 8 : 4;
    EXL2B_REQUIRE(head_dim == 64 || head_dim == 128, "head_dim %d not supported (64 or 128)", head_dim);
    EXL2B_REQUIRE(num_heads % num_kv_heads == 0, "bad GQA ratio");
    EXL2B_REQUIRE(q_len >= 1 && q_len <= AQ_MAX_QLEN, "q_len %d outside the decode regime (1..%d)", q_len, AQ_MAX_QLEN);
    AttnQ4Params P = {};
    P.q = (const half*)q; P.k_new = (const half*)k_new; P.v_new = (const half*)v_new;
    P.k_q = k_cache; P.k_s = (half*)k_scales; P.v_q = v_cache; P.v_s = (half*)v_scales;
    P.cache_seqlens = cache_seqlens; P.block_table = block_table; P.out = (half*)out;
    P.q_len = q_len; P.H = num_heads; P.KVH = num_kv_heads; P.hd = head_dim;
    P.page_size = page_size; P.pages_per_seq = pages_per_seq;
    P.max_ctx = page_size * pages_per_seq;
    P.scale_log2 = softmax_scale * 1.4426950408889634f;
    if (out_consumer) {
        QMatrix* oc = (QMatrix*)out_consumer;
        EXL2B_REQUIRE(oc->v.layout == LAYOUT_TC && oc->v.K == num_heads * head_dim, "out_consumer does not take the attention output");
        EXL2B_REQUIRE(batch * q_len <= 8, "chained attention output needs at most 8 rows");
        int rc = qmatrix_chain_buffers(oc);
        if (rc) return rc;
        P.out_xp = oc->xp_buf;
        P.out_invperm = oc->invperm;
        P.out_plain = (batch * q_len == 1 && gemv_i8_enabled()) ? 1 : 0;      // the single-row GEMV reads a plain fp16 row
    }
    if (rope_style != 0 && rope_sin && rope_cos) {
        EXL2B_REQUIRE(sincos_size == head_dim, "fused RoPE needs sincos_size == head_dim (partial rotary: apply rope_ first)");
        P.rope_sin = (const half*)rope_sin;
        P.rope_cos = (const half*)rope_cos;
        P.rope_neox = rope_style == 2;
        P.sincos_size = sincos_size;
    }
    int dev = 0;
    EXL2B_CUDA(cudaGetDevice(&dev));
    if (dev >= 0 && dev < 64) {
        if (!g_attn_err[dev]) {
            EXL2B_CUDA(cudaMalloc(&g_attn_err[dev], sizeof(int32_t)));
            EXL2B_CUDA(cudaMemset(g_attn_err[dev], 0, sizeof(int32_t)));
        }
        P.err = g_attn_err[dev];
    }
    // split-KV: only for single-query decode over caches long enough to need it; grid.z CTAs per (head, sequence)
    int nsplit = 1;
    if (q_len == 1 && P.max_ctx > 2 * AQ_SPLIT_MIN) {
        const int sms = device_sm_count(dev);
        const int by_ctx = (P.max_ctx + AQ_SPLIT_MIN - 1) / AQ_SPLIT_MIN;
        const int by_sms = std::max(1, (2 * sms) / std::max(1, num_heads * batch));
        nsplit = std::max(1, std::min(std::min(by_ctx, by_sms), 16));
    }
    static float* g_ws[64] = {nullptr};
    static unsigned int* g_cnt[64] = {nullptr};
    static size_t g_ws_floats[64] = {0}, g_cnt_n[64] = {0};
    if (nsplit > 1) {
        EXL2B_REQUIRE(dev >= 0 && dev < 64, "bad device");
        const size_t need = (size_t)batch * num_heads * nsplit * (head_dim + 2), need_c = (size_t)batch * num_heads;
        if (g_ws_floats[dev] < need) {
            if (g_ws[dev]) cudaFree(g_ws[dev]);
            EXL2B_CUDA(cudaMalloc(&g_ws[dev], need * sizeof(float)));
            g_ws_floats[dev] = need;
        }
        if (g_cnt_n[dev] < need_c) {
            if (g_cnt[dev]) cudaFree(g_cnt[dev]);
            EXL2B_CUDA(cudaMalloc(&g_cnt[dev], need_c * sizeof(unsigned)));
            EXL2B_CUDA(cudaMemset(g_cnt[dev], 0, need_c * sizeof(unsigned)));
            g_cnt_n[dev] = need_c;
        }
        P.ws = g_ws[dev];
        P.cnt = g_cnt[dev];
    }
    P.nsplit = nsplit;
    {
        P.dbg = exl2b::g_dbg ? exl2b::g_dbg + 32 * (exl2b::g_dbg_slot++ % 64) : nullptr;
        P.dbg_cta = 0;
    }
    const int sc_len = nsplit > 1 ? std::max(AQ_SPLIT_MIN, (P.max_ctx + nsplit) / nsplit) + 8 : P.max_ctx + q_len;
    const int hd = head_dim;
    P.sc_len = sc_len;
    // cached rows beyond the staged window: streamed through a ring of 4 sub-chunks (128 positions at Q4) when the cache is long;
    // the ring takes the place of half the staged window, so the CTA keeps the footprint that lets it share an SM with one GEMV
    // CTA (a first version that ADDED the ring lost that co-residency).  The ring pays once a CTA has thousands of positions;
    // below, the larger window wins.  The host only knows the cache's capacity:
    P.ring_slots = (P.max_ctx > 8192) ? AQ_RING : 0;
    // The window and the ring are sized in BYTES: every format stages at most the bytes of Q4's AQ_STAGE (or AQ_STAGE / 2 with
    // the ring) positions, in whole multiples of 64 positions, so no format needs more shared memory than Q4: Q8 stages 256
    // (128) positions, Q6 320 (128).  Ring sub-chunks hold the bytes of 128 Q4 rows of the wider of K and V (64 at 8 bits).
    const int rowk = hd * kb / 8, rowv = hd * vb / 8, nsc = hd / 32;
    const int window = P.ring_slots ? AQ_STAGE / 2 : AQ_STAGE;
    P.stage = (int)((size_t)window * (hd + 4 * nsc) / (size_t)(rowk + rowv + 4 * nsc)) / 64 * 64;
    const int sub = AQ_SUB * 4 / std::max(kb, vb);
    const size_t smem = (size_t)((hd / 32) * 36 + AQ_WARPS * hd + 2 * AQ_WARPS) * 4 + (size_t)(hd / 32) * (80 + 8) + AQ_MAX_QLEN * (rowk + rowv) + 2 * AQ_MAX_QLEN * (hd / 32) * 2 +
                        (size_t)2 * AQ_MAX_QLEN * hd * 4 + (size_t)((pages_per_seq + 3) & ~3) * 4 + (size_t)((sc_len + 3) & ~3) * 4 +
                        (size_t)P.stage * (rowk + rowv) + (size_t)P.stage * nsc * 2 * 2 +
                        (P.ring_slots ? (size_t)AQ_RING * sub * (std::max(rowk, rowv) + nsc * 2) : 0);
    EXL2B_REQUIRE(smem <= 200 * 1024, "context of %d tokens does not fit the score buffer", P.max_ctx);
    static bool attr_set[64] = {false};
    if (!attr_set[dev]) {
        int rc = attn_q_set_smem<4, 4>();
        if (!rc) rc = attn_q_set_smem<8, 4>();
        if (!rc) rc = attn_q_set_smem<8, 8>();
        if (rc) return rc;
        attr_set[dev] = true;
    }
    static unsigned int* slot_cnts[64] = {nullptr};
    static std::atomic<unsigned> launch_seq{0};
    if (!slot_cnts[dev]) {
        EXL2B_CUDA(cudaMalloc(&slot_cnts[dev], 128 * sizeof(unsigned int)));
        EXL2B_CUDA(cudaMemset(slot_cnts[dev], 0, 128 * sizeof(unsigned int)));
    }
    P.slot_cnt = slot_cnts[dev] + (launch_seq.fetch_add(1) % 127u);
    P.batch = batch;
    P.busy_ctas = num_heads * batch * nsplit;
    dim3 grid(slot_holders_disabled() ? P.busy_ctas : std::max(P.busy_ctas, device_sm_count(dev)));
    if (wbits == 4) return attn_q_launch<4, 4>(head_dim, grid, smem, (cudaStream_t)stream, P);
    if (wbits == 6) return attn_q_launch<8, 4>(head_dim, grid, smem, (cudaStream_t)stream, P);
    return attn_q_launch<8, 8>(head_dim, grid, smem, (cudaStream_t)stream, P);
}
