// Decode attention straight over the Q4 / Q6 / Q8 K/V cache: quantise-and-append the new rows, attend, in ONE kernel.
//
// The reference runs, per layer and per step (exllamav2/attn.py:560-613, cache.py:472-556):
//     q_to_fp16_kv over the WHOLE live cache -> flash_attn_with_kvcache on the fp16 temp -> fp16_to_q_kv of the new rows
// i.e. it expands every cached nibble to fp16 in HBM and reads it back.  Here the cache is consumed as stored
// (0.5 B + 1/16 B per value):
//   * the cache holds y = H32 x per 64-value unit (unnormalised Hadamard on the even / odd interleaved 32-vectors,
//     kv_format.cuh), quantised to 4 bits with an fp16 scale per 32 consecutive values.  H is symmetric and H H = 32 I, so
//         q . x = (H q) . y / 32            sum_s p_s x_s = H (sum_s p_s y_s) / 32
//     the query is rotated ONCE, scores and the P V sum are formed on the stored (rotated) values, and the output is
//     rotated back ONCE -- no per-position butterflies.
//   * the kernel is templated on the element widths of keys (KB) and values (VB): (4, 4) is the Q4 cache, (8, 4) Q6 and
//     (8, 8) Q8 (kvcache.cu).  An 8-bit row holds value e of a 32-value block at byte e, one fp16 scale per block as in Q4.
//   * the q_len new K/V rows are quantised with the cache format's own arithmetic (kv_format.cuh kv_quantise, same bits as
//     fp16_to_q_kv and the reference) and written to the paged cache by one designated CTA per kv head.  The step that appends
//     them attends them UNQUANTISED (fp16 values, rotated in fp32), exactly like the reference, where
//     flash_attn_with_kvcache sees the fp16 rows and the cache only quantises them afterwards (attn.py:602-621).
// One CTA per (head, sequence); decode regime (q_len <= 8).  The kernel runs as phases over a per-CTA context (AttnCta):
// prologue and staging, new-row quantisation and query rotation, scores, softmax, P V, append, end of the query.
#include <algorithm>
#include <map>
#include <mutex>

#include "gemv.cuh"
#include "gemv_i8.cuh"
#include "kv_format.cuh"
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
    int out_tw;             // token slots of that layout: the consumer launch's wgmma tile (tc_tile of batch * q_len)
    int32_t* err;           // sticky device flag: bit 0 = a sequence ran past its page table (nothing appended, no output)
    // split-KV (long contexts, q_len == 1): grid.z CTAs share one (head, sequence); each attends a contiguous chunk of positions
    // and leaves (max, sum, unnormalised rotated output) in `ws`; the last to arrive (counter) merges.  Chunks are at least
    // AQ_SPLIT_MIN positions, so short contexts use one CTA and never touch the workspace.
    int sc_len;             // floats of the score buffer
    int stage;              // cached positions per CTA copied to shared memory before the dependency wait (the bytes of AQ_STAGE Q4 rows; half with the ring)
    int ring_slots;         // long contexts: cached rows beyond the staged window stream through a ring of sub-chunks (aq_sub) (0: loads from global)
    int batch;              // grid: one CTA per (head, sequence, split), flattened on x, padded to one CTA per SM with slot holders
    int busy_ctas;          //   = H * batch * nsplit
    unsigned int* slot_cnt; // CTAs of this launch that are done (self-resetting, common.cuh slot_release)
    int nsplit;
    float* ws;              // [batch][H][nsplit][hd + 2]
    unsigned int* cnt;      // [batch][H]
    unsigned long long* dbg;   // optional globaltimer stamps of CTA (dbg_cta, 0, 0) (exl2b_debug_set): 0 start, 1 cache rows requested,
    int dbg_cta;               //   2 dependency wait over, 3 new rows quantised / query rotated, 4 scores + max, 5 P V done; 6 / 7 grid span;
                               //   dbg[10] counts the CTAs that took staged_pass (all_staged)
    int pass_len;              // attn_q4_passes_kernel: positions per pass (= sc_len); 0 for attn_q4_kernel
};
constexpr int AQ_SPLIT_MIN = 512;
constexpr int AQ_SUB = 128;            // positions per sub-chunk of the streaming ring (long contexts)
constexpr int AQ_RING = 4;             // sub-chunks in flight
constexpr int AQ_STAGE = 512;          // cached positions per CTA staged in shared memory before the dependency wait (Q4; the
                                       // other formats stage the same number of BYTES, host side)
constexpr int AQ_SMEM_MAX = 200 * 1024;     // dynamic shared memory a launch may use
// Single-token decode over a cache whose whole-chunk score buffer does not fit AQ_SMEM_MAX walks each CTA's positions in
// passes (attn_q4_passes_kernel).  The pass length is chosen so that the CTA still shares an SM with one batch-1 GEMV CTA:
// 228 KB per SM - 111 KB for the GEMV CTA (gemv_i8.cu) - 1 KB reserved per CTA for each of the two - 1 KB for this kernel's
// static shared memory and slack = 114 KB.  A page table too large for that still runs, with passes of AQ_PASS_MIN positions
// and without the co-residency; only a page table that leaves no room for AQ_PASS_MIN positions under AQ_SMEM_MAX is refused.
constexpr int AQ_PASS_SMEM = 114 * 1024;
constexpr int AQ_PASS_MIN = 512;
constexpr int AQ_PASS_ALIGN = 256;     // pass lengths are multiples of 256 positions (whole pages at the default page size):
                                       // a multiple of every ring sub-chunk and score pass
constexpr int AQ_QPAD = 36;            // floats per 32-value block of the rotated query (bank-staggered: 4 blocks, 4 threads per row)
constexpr int AQ_QIB = 80;             // bytes per 32-value block of the integer query operands (64 used; bank-staggered like QPAD)

__host__ __device__ constexpr int aq_sub(int kb, int vb) { return AQ_SUB * 4 / (kb > vb ? kb : vb); }   // ring sub-chunk positions: the Q4 sub-chunk's bytes

// dynamic shared-memory map of a CTA (byte offsets) -- one definition for the kernel and the host that sizes the launch
struct AttnSmem {
    uint32_t qrot, qi, qsum, qscl, red, wred, new_q, new_s, new_y, pages, sc, kst, vst, ksst, vsst, rq, rs, total;
};
__host__ __device__ inline AttnSmem attn_smem_map(int hd, int kb, int vb, int pages_per_seq, int sc_len, int stage, bool ring) {
    const uint32_t nsc = hd / 32, rowk = hd * kb / 8, rowv = hd * vb / 8, sub = aq_sub(kb, vb);
    AttnSmem m;
    m.qrot = 0;                                                 // [NSC][QPAD]  rotated query, fp32
    m.qi = m.qrot + nsc * AQ_QPAD * 4;                          // [NSC][QIB]   16-bit query as dp4a byte operands (rotate_q)
    m.qsum = m.qi + nsc * AQ_QIB;                               // [NSC]        sum of a block's 16-bit values
    m.qscl = m.qsum + nsc * 4;                                  // [NSC]        its power-of-two scale
    m.red = m.qscl + nsc * 4;                                   // [AQ_WARPS][HD]  per-warp P V sums
    m.wred = m.red + AQ_WARPS * hd * 4;                         // [2 * AQ_WARPS]  per-warp max, then sum
    m.new_q = m.wred + 2 * AQ_WARPS * 4;                        // [AQ_MAX_QLEN][ROWBK], then [AQ_MAX_QLEN][ROWBV]
    m.new_s = m.new_q + AQ_MAX_QLEN * (rowk + rowv);            // [2][AQ_MAX_QLEN][NSC]
    m.new_y = m.new_s + 2 * AQ_MAX_QLEN * nsc * 2;              // [2][AQ_MAX_QLEN][HD] rotated, unquantised new rows
    m.pages = m.new_y + 2 * AQ_MAX_QLEN * hd * 4;               // [pages_per_seq]
    m.sc = m.pages + ((pages_per_seq + 3) & ~3) * 4;            // [sc_len] scores, then softmax weights
    m.kst = m.sc + ((sc_len + 3) & ~3) * 4;                     // [stage][ROWBK]  staged cached K rows
    m.vst = m.kst + stage * rowk;                               // [stage][ROWBV]
    m.ksst = m.vst + stage * rowv;                              // [stage][NSC]
    m.vsst = m.ksst + stage * nsc * 2;
    m.rq = m.vsst + stage * nsc * 2;                            // [AQ_RING][SUB][ROWB]  streaming ring (K, then V), if `ring`
    m.rs = m.rq + AQ_RING * sub * (rowk > rowv ? rowk : rowv);  // [AQ_RING][SUB][NSC]
    m.total = ring ? m.rs + AQ_RING * sub * nsc * 2 : m.rq;
    return m;
}

// A cached row: straight from the cache, or from its copy in shared memory.  Cached K/V rows and their scales are read once per
// step (every copy and load of them below is evict-first in L2, common.cuh); the rows this step appends, the page table,
// sin / cos, q / k / v and the split-KV scratch keep the default policy.
template <bool GLOBAL, typename T>
__device__ __forceinline__ T ld_rows(const T* p) {
    if constexpr (GLOBAL) return ldg_ef(p);
    else return *p;
}

// the sin / cos pair that rotates one lane's half2 of 64-value unit `un` of a head row at position pos (fused RoPE)
struct RopeCs {
    half2 c, s;
};
template <int HD>
__device__ __forceinline__ RopeCs rope_cs(int un, int lane, const AttnQ4Params& P, int pos) {
    // NeoX pairs element j with j + HD / 2: HD == 128, the other unit at the same lane; HD == 64, lane ^ 16
    const int col = !P.rope_neox ? un * 64 + 2 * lane : HD == 128 ? 2 * lane : 2 * (lane & 15);
    return {*reinterpret_cast<const half2*>(P.rope_cos + (size_t)pos * P.sincos_size + col),
            *reinterpret_cast<const half2*>(P.rope_sin + (size_t)pos * P.sincos_size + col)};
}

// one half2 (elements un*64 + 2*lane, +1) of a head row, rotated with `cs` (rope_cs) if RoPE is fused.  Warp-uniform call.
template <int HD>
__device__ __forceinline__ half2 load_roped(const half* __restrict__ row, int un, int lane, const AttnQ4Params& P, const RopeCs& cs) {
    const half2 v = reinterpret_cast<const half2*>(row + un * 64)[lane];
    if (!P.rope_sin) return v;
    if (P.rope_neox) {
        half2 o;
        bool first;
        if constexpr (HD == 128) {            // partner element j + 64 lives in the other 64-value unit, same lane
            o = reinterpret_cast<const half2*>(row + (un ^ 1) * 64)[lane];
            first = (un == 0);
        } else {                              // HD == 64: partner j + 32 is lane ^ 16
            o = __shfl_xor_sync(0xffffffffu, v, 16);
            first = lane < 16;
        }
        if (first) return __hfma2(v, cs.c, __hmul2(o, __hneg2(cs.s)));      // l' = l c + half(r * -s)
        return __hfma2(v, cs.c, __hmul2(o, cs.s));                            // r' = r c + half(l * s)
    }
    half2 s01 = cs.s;
    uint32_t sb = *reinterpret_cast<uint32_t*>(&s01) ^ (1u << 15);        // (-sin[i], +sin[i+1])
    s01 = *reinterpret_cast<half2*>(&sb);
    return __hfma2(__lowhigh2highlow(v), s01, __hmul2(v, cs.c));
}

// (nibble - 8) as fp32 without I2F: 0x4B000000 | n is the float 2^23 + n
__device__ __forceinline__ float nib_f(uint32_t n) { return __uint_as_float(0x4B000000u | n) - 8388616.0f; }
// (byte - 128) as fp32, same trick
__device__ __forceinline__ float byte_f(uint32_t n) { return __uint_as_float(0x4B000000u | n) - 8388736.0f; }

// every exit of a working CTA: count it (slot holders of the launch leave when all working CTAs have)
__device__ __forceinline__ void cta_exit(const AttnQ4Params& P) {
    if (threadIdx.x == 0) slot_release(P.slot_cnt);
}

// One working CTA: its (head, sequence, split), its share of the positions and its shared memory.  The member functions are
// the kernel's phases, in the order attn_q4_kernel runs them.
template <int HD, int KB, int VB>
struct AttnCta {
    static_assert((KB == 4 || KB == 8) && (VB == 4 || VB == 8), "element widths are 4 or 8 bits");
    static constexpr int ROWBK = HD * KB / 8;      // packed bytes per (position, kv head): keys
    static constexpr int ROWBV = HD * VB / 8;      //   values
    static constexpr int ROWB = ROWBK > ROWBV ? ROWBK : ROWBV;     // one ring slot position (keys, then values)
    static constexpr int SUB = aq_sub(KB, VB);
    static constexpr int NSC = HD / 32;            // scales per (position, kv head)
    static constexpr int VEC = HD / 32;            // values per lane in the dims-on-lanes phase
    static constexpr int UNITS = HD / 64;
    static constexpr int TPR = NSC, RPP = AQ_THREADS / TPR;      // scores: NSC threads per position (one 32-value block + scale each)
    static constexpr int KW = KB / 4;              // uint4 words per 32-value key block
    static constexpr uint32_t KFILL = KB == 4 ? 0x88888888u : 0x80808080u;      // a zero block (never scored: keeps registers defined)

    const AttnQ4Params& P;
    float* qrot;
    uint8_t* qi;
    int* qsum;
    float* qscl;
    float* red;
    float* wred;
    uint8_t* new_q;
    half* new_s;
    float* new_y;
    int* pages_s;
    float* sc;
    uint8_t *kst, *vst;
    half *ksst, *vsst;
    uint8_t* rq;
    half* rs;
    int h, b, z, tid, warp, lane, group, kvh, kblk, krow;
    int seqlen, ns_act, p_lo, p_hi, c_hi, n_st, ntail;
    const int* bt;                                 // the sequence's page table: global until the prologue has copied it
    RopeCs cs0;                                    // fused RoPE: sin / cos at position seqlen of this warp's rope_unit() (load_static)

    __device__ __forceinline__ AttnCta(const AttnQ4Params& P_, uint8_t* smem) : P(P_) {
        const AttnSmem m = attn_smem_map(HD, KB, VB, P.pages_per_seq, P.sc_len, P.stage, true);
        qrot = reinterpret_cast<float*>(smem + m.qrot);
        qi = smem + m.qi;
        qsum = reinterpret_cast<int*>(smem + m.qsum);
        qscl = reinterpret_cast<float*>(smem + m.qscl);
        red = reinterpret_cast<float*>(smem + m.red);
        wred = reinterpret_cast<float*>(smem + m.wred);
        new_q = smem + m.new_q;
        new_s = reinterpret_cast<half*>(smem + m.new_s);
        new_y = reinterpret_cast<float*>(smem + m.new_y);
        pages_s = reinterpret_cast<int*>(smem + m.pages);
        sc = reinterpret_cast<float*>(smem + m.sc);
        kst = smem + m.kst;
        vst = smem + m.vst;
        ksst = reinterpret_cast<half*>(smem + m.ksst);
        vsst = reinterpret_cast<half*>(smem + m.vsst);
        rq = smem + m.rq;
        rs = reinterpret_cast<half*>(smem + m.rs);
        h = (int)blockIdx.x % P.H;
        b = ((int)blockIdx.x / P.H) % P.batch;
        z = (int)blockIdx.x / (P.H * P.batch);
        tid = threadIdx.x;
        warp = tid >> 5;
        lane = tid & 31;
        group = P.H / P.KVH;
        kvh = h / group;
        kblk = tid & (TPR - 1);
        krow = tid / TPR;
    }

    // the cache row of position p of this sequence and kv head
    __device__ __forceinline__ size_t row(int p) const {
        const int page = bt[p / P.page_size];
        return ((size_t)page * P.page_size + p % P.page_size) * P.KVH + kvh;
    }

    // ---- prologue, before the dependency wait: everything that only touches state written by EARLIER steps / layers -- the
    //      sequence length, the page table and the cached rows (this layer's cache was last written one decode step ago; the
    //      kernel in front of us in the stream, the Q|K|V projection, writes none of it).  False: the CTA has nothing to do.
    __device__ __forceinline__ bool prologue() {
        seqlen = P.cache_seqlens[b];
        if (seqlen < 0 || seqlen + P.q_len > P.max_ctx) {      // the page table / score buffer end here: refuse instead of corrupting
            if (tid == 0 && P.err) atomicOr(P.err, 1);
            return false;
        }
        bt = P.block_table + (size_t)b * P.pages_per_seq;
        // this CTA's share of the positions (the whole context unless split-KV is active and the context is long)
        ns_act = 1;
        p_lo = 0;
        p_hi = seqlen + P.q_len;
        if (P.nsplit > 1) {
            const int n_all = seqlen + 1;
            ns_act = min(P.nsplit, max(1, (n_all + AQ_SPLIT_MIN - 1) / AQ_SPLIT_MIN));
            if (z >= ns_act) return false;
            const int chunk = (n_all + ns_act - 1) / ns_act;
            p_lo = z * chunk;
            p_hi = min(n_all, p_lo + chunk);
        }
        c_hi = min(p_hi, seqlen);          // cached rows of this CTA: [p_lo, c_hi)
        // the first P.stage of them are copied to shared memory with cp.async (no registers held across the wait): K / V elements
        // [pos][ROWBK] / [pos][ROWBV] and their fp16 scales [pos][NSC]
        n_st = max(0, min(c_hi - p_lo, P.stage));
        constexpr int CHK = ROWBK / 16, CHV = ROWBV / 16, CH = CHK > CHV ? CHK : CHV;      // 16-byte chunks per row
        for (int idx = tid; idx < n_st * CH; idx += AQ_THREADS) {
            const int pos = idx / CH, ch = idx - pos * CH;
            const size_t r = row(p_lo + pos);
            if (ch < CHK) cp_async16_ef(smem_addr(kst + pos * ROWBK + ch * 16), P.k_q + r * ROWBK + ch * 16);
            if (ch < CHV) cp_async16_ef(smem_addr(vst + pos * ROWBV + ch * 16), P.v_q + r * ROWBV + ch * 16);
        }
        for (int pos = tid; pos < n_st; pos += AQ_THREADS) {
            const size_t r = row(p_lo + pos);
            cp_async_small_ef<NSC * 2>(smem_addr(ksst + pos * NSC), P.k_s + r * NSC);
            cp_async_small_ef<NSC * 2>(smem_addr(vsst + pos * NSC), P.v_s + r * NSC);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        for (int i = tid; i < P.pages_per_seq; i += AQ_THREADS) pages_s[i] = bt[i];
        bt = pages_s;
        ntail = ring_chunks();
        return true;
    }
    // operands of the phases after the dependency wait that the Q|K|V launch does not write, fetched just before the wait
    // (not in the prologue: registers held across staged_pass's first run spill).  The fused-RoPE sin / cos pair is loaded;
    // the o_proj rows store_out writes are only prefetched into L2, so that they hold no register until the store.
    __device__ __forceinline__ void load_static() {
        cs0 = P.rope_sin ? rope_cs<HD>(rope_unit(), lane, P, seqlen) : RopeCs{};
        if (P.out_invperm && warp < UNITS && lane == 0)
            asm volatile("prefetch.global.L2 [%0];" ::"l"(P.out_invperm + h * HD + warp * 64));
    }
    // the 64-value unit whose RoPE the warp applies first (new_rows_and_first_query): the last UNITS warps rotate the query,
    // the first ones quantise the new rows, job = warp (key rows are jobs 0 .. UNITS - 1)
    __device__ __forceinline__ int rope_unit() const {
        return warp >= AQ_WARPS - UNITS ? warp - (AQ_WARPS - UNITS) : warp % UNITS;
    }
    // unit un of a head row at position seqlen + i, rotated if RoPE is fused (sin / cos from the prologue where they match)
    __device__ __forceinline__ half2 roped(const half* row, int un, int i) const {
        const bool pre = !P.rope_sin || (i == 0 && un == rope_unit());
        return load_roped<HD>(row, un, lane, P, pre ? cs0 : rope_cs<HD>(un, lane, P, seqlen + i));
    }
    // ring sub-chunks of the cached rows [p_lo + n_st, c_hi) (0 without the ring)
    __device__ __forceinline__ int ring_chunks() const {
        return (P.ring_slots && c_hi > p_lo + n_st) ? (c_hi - (p_lo + n_st) + SUB - 1) / SUB : 0;
    }

    // ---- attn_q4_passes_kernel: the phases below walk [p_lo, n_ctx) with the scores in sc[p - p_lo], the staged window
    //      [p_lo, p_lo + n_st) and the ring over [p_lo + n_st, c_hi).  Pass [lo, hi) of the CTA's share points them at its
    //      positions; only the first pass has the staged window (nst), later ones stream every cached row through the ring.
    __device__ __forceinline__ void begin_pass(int lo, int hi, int nst) {
        p_lo = lo;
        c_hi = min(hi, seqlen);
        n_st = nst;
        ntail = ring_chunks();
    }

    // ---- query i, 64-value unit un, on one warp: qrot = H q * (softmax_scale * log2 e / 32), and its integer operands
    __device__ __forceinline__ void rotate_q(int i, int un) {
        const half2 qh = roped(P.q + (((size_t)b * P.q_len + i) * P.H + h) * HD, un, i);
        float2 w = hadamard32_f(__half22float2(qh), lane);
        const float f = P.scale_log2 * (1.0f / 32.0f);
        const int e = un * 64 + 2 * lane;
        w.x *= f;
        w.y *= f;
        qrot[(e >> 5) * AQ_QPAD + (e & 31)] = w.x;
        qrot[(e >> 5) * AQ_QPAD + (e & 31) + 1] = w.y;
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
            uint8_t* qb = qi + blk * AQ_QIB + j * 16 + m;          // word order per j: even-high, even-low, odd-high, odd-low
            qb[0] = (uint8_t)(q0 >> 8);
            qb[4] = (uint8_t)q0;
            qb[8] = (uint8_t)(q1 >> 8);
            qb[12] = (uint8_t)q1;
        } else {
            // 8-bit keys: word w of a block holds values 4w..4w+3 in byte order; per pair of words j = w / 2 the 16 bytes are
            // high(w = 2j), low(2j), high(2j + 1), low(2j + 1).  This lane's values 2 l16, 2 l16 + 1 sit in word l16 / 2.
            const int w8 = l16 >> 1;
            uint8_t* qb = qi + blk * AQ_QIB + (w8 >> 1) * 16 + (w8 & 1) * 8 + (l16 & 1) * 2;
            qb[0] = (uint8_t)(q0 >> 8);
            qb[1] = (uint8_t)(q1 >> 8);
            qb[4] = (uint8_t)q0;
            qb[5] = (uint8_t)q1;
        }
        if (l16 == 0) {
            qsum[blk] = sum;
            qscl[blk] = amax > 0.f ? __uint_as_float((ef - 14u) << 23) : 0.f;
        }
    }

    // ---- quantise the new rows (kv_format.cuh) on the first warps, keep them in shared memory; at the same time the LAST
    //      warps rotate the first query
    __device__ __forceinline__ void new_rows_and_first_query() {
        if (warp >= AQ_WARPS - UNITS) rotate_q(0, warp - (AQ_WARPS - UNITS));
        const int n_jobs = 2 * P.q_len * UNITS;
        for (int job = (warp >= AQ_WARPS - UNITS && n_jobs <= AQ_WARPS - UNITS) ? n_jobs : warp; job < n_jobs; job += AQ_WARPS) {
            const int kv = job / (P.q_len * UNITS), r = job - kv * P.q_len * UNITS;
            const int i = r / UNITS, un = r - i * UNITS;
            const half* src = (kv ? P.v_new : P.k_new) + (((size_t)b * P.q_len + i) * P.KVH + kvh) * HD;
            half2 w2 = kv ? reinterpret_cast<const half2*>(src + un * 64)[lane] : roped(src, un, i);
            {
                const float2 y = hadamard32_f(__half22float2(w2), lane);
                new_y[(kv * AQ_MAX_QLEN + i) * HD + un * 64 + 2 * lane] = y.x;
                new_y[(kv * AQ_MAX_QLEN + i) * HD + un * 64 + 2 * lane + 1] = y.y;
            }
            w2 = hadamard32_h(w2, lane);
            uint8_t* nq = new_q + (kv ? AQ_MAX_QLEN * ROWBK + i * ROWBV : i * ROWBK);
            half* ns = new_s + (kv * AQ_MAX_QLEN + i) * NSC + un * 2 + (lane >> 4);
            if ((kv ? VB : KB) == 4) {
                const KvCodes c = kv_quantise<4>(w2);
                nq[un * 32 + lane] = (uint8_t)(c.q0 | (c.q1 << 4));
                if ((lane & 15) == 0) *ns = c.scale;
            } else {
                const KvCodes c = kv_quantise<8>(w2);
                reinterpret_cast<uint16_t*>(nq + un * 64)[lane] = (uint16_t)(c.q0 | (c.q1 << 8));
                if ((lane & 15) == 0) *ns = c.scale;
            }
        }
    }

    // sub-chunk t of the cached rows beyond the staged window -> ring slot t % AQ_RING (one cp.async group per call, possibly
    // empty); rows of RB bytes (keys, then values) at a pitch of ROWB
    template <int RB>
    __device__ __forceinline__ void ring_issue(int t, const uint8_t* gq, const half* gs) const {
        constexpr int CH = RB / 16;
        const int base = p_lo + n_st + t * SUB, cnt = min(SUB, c_hi - base), slot = t & (AQ_RING - 1);
        for (int idx = tid; idx < cnt * CH; idx += AQ_THREADS) {
            const int pos = idx / CH, ch = idx - pos * CH;
            cp_async16_ef(smem_addr(rq + (slot * SUB + pos) * ROWB + ch * 16), gq + row(base + pos) * RB + ch * 16);
        }
        for (int pos = tid; pos < cnt; pos += AQ_THREADS)
            cp_async_small_ef<NSC * 2>(smem_addr(rs + (slot * SUB + pos) * NSC), gs + row(base + pos) * NSC);
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    // long context: the cached rows beyond the staged window stream through the ring, AQ_RING sub-chunks in flight;
    // consume(base, rows, scales) reads the sub-chunk of positions from base on out of its slot
    template <int RB, typename F>
    __device__ __forceinline__ void ring_pass(const uint8_t* gq, const half* gs, F&& consume) const {
        __syncthreads();                                  // (every thread is done with the ring's previous contents)
        for (int t = 0; t < AQ_RING; ++t) ring_issue<RB>(t, gq, gs);
        for (int t = 0; t < ntail; ++t) {
            asm volatile("cp.async.wait_group %0;" ::"n"(AQ_RING - 1) : "memory");
            __syncthreads();
            const int slot = t & (AQ_RING - 1);
            consume(p_lo + n_st + t * SUB, rq + slot * SUB * ROWB, rs + slot * SUB * NSC);
            __syncthreads();
            ring_issue<RB>(t + AQ_RING, gq, gs);
        }
    }

    // ---- scores: NSC threads per position, each its 32-value block (kblk) of the (rotated) row against qrot
    struct KeyBlock {
        uint4 w[KW];
        uint32_t s;       // fp16 scale bits
    };
    __device__ __forceinline__ static KeyBlock key_none() {
        KeyBlock k;
#pragma unroll
        for (int u = 0; u < KW; ++u) k.w[u] = make_uint4(KFILL, KFILL, KFILL, KFILL);
        k.s = 0u;
        return k;
    }
    // this thread's block of a cached key row and its scale: in shared memory (staged window, ring), or (GLOBAL) in the cache
    template <bool GLOBAL>
    __device__ __forceinline__ KeyBlock key_block(const uint8_t* rowq, const half* rows) const {
        KeyBlock k;
#pragma unroll
        for (int u = 0; u < KW; ++u) k.w[u] = ld_rows<GLOBAL>(reinterpret_cast<const uint4*>(rowq) + kblk * KW + u);
        k.s = ld_rows<GLOBAL>(reinterpret_cast<const unsigned short*>(rows) + kblk);
        return k;
    }
    __device__ __forceinline__ KeyBlock key_global(int p) const {
        const size_t r = row(p);
        return key_block<true>(P.k_q + r * ROWBK, P.k_s + r * NSC);
    }

    // score of one 32-value block of a cached row (one fp16 scale) against its block of the rotated query, all in integers (dp4a),
    // one fp32 multiply at the end.  4 bits: sum_d (nib_d - 8) q_d = sum nib q - 8 sum q, dp4a on the masked words.
    // 8 bits: sum_d (b_d - 128) q_d = sum b q - 128 sum q, dp4a on the stored words as they are.  The offset is removed with the
    // block's query sum (one multiply-add per block, shared with the 4-bit path) rather than by flipping every byte's top bit and
    // using signed dp4a (one extra logic op per word, 8 per block).
    __device__ __forceinline__ float score_blk(const KeyBlock& k) const {
        const uint8_t* qb = qi + kblk * AQ_QIB;
        int v;
        if constexpr (KB == 4) {
            const uint32_t ww[4] = {k.w[0].x, k.w[0].y, k.w[0].z, k.w[0].w};
            int a0 = 0, a1 = 0, a2 = 0, a3 = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint4 qo = *reinterpret_cast<const uint4*>(qb + j * 16);
                const uint32_t lo = ww[j] & 0x0f0f0f0fu, hi = ww[j] & 0xf0f0f0f0u;
                a0 = dp4a_us(lo, qo.x, a0);          // unsigned nibbles x signed high bytes
                a1 = dp4a_uu(lo, qo.y, a1);          // unsigned x unsigned low bytes
                a2 = dp4a_us(hi, qo.z, a2);
                a3 = dp4a_uu(hi, qo.w, a3);
            }
            v = ((a0 << 8) + a1) + (((a2 << 8) + a3) >> 4) - 8 * qsum[kblk];
        } else {
            const uint32_t ww[8] = {k.w[0].x, k.w[0].y, k.w[0].z, k.w[0].w, k.w[1].x, k.w[1].y, k.w[1].z, k.w[1].w};
            int a0 = 0, a1 = 0, a2 = 0, a3 = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint4 qo = *reinterpret_cast<const uint4*>(qb + j * 16);
                a0 = dp4a_us(ww[2 * j], qo.x, a0);          // unsigned bytes x signed high bytes
                a1 = dp4a_uu(ww[2 * j], qo.y, a1);          // unsigned x unsigned low bytes
                a2 = dp4a_us(ww[2 * j + 1], qo.z, a2);
                a3 = dp4a_uu(ww[2 * j + 1], qo.w, a3);
            }
            v = ((a0 + a2) << 8) + (a1 + a3) - 128 * qsum[kblk];
        }
        return __half2float(__ushort_as_half((unsigned short)k.s)) * qscl[kblk] * (float)v;
    }

    // this thread's block of the score of new row i (appended by this step): fp16 values, rotated in fp32
    __device__ __forceinline__ float score_new(int i) const {
        const float4* y4 = reinterpret_cast<const float4*>(new_y + i * HD + kblk * 32);
        const float4* q4 = reinterpret_cast<const float4*>(qrot + kblk * AQ_QPAD);
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float4 a = q4[j], c = y4[j];
            s0 = fmaf(a.x, c.x, s0);
            s1 = fmaf(a.y, c.y, s1);
            s2 = fmaf(a.z, c.z, s2);
            s3 = fmaf(a.w, c.w, s3);
        }
        return (s0 + s1) + (s2 + s3);
    }

    // score of position p (warp-uniform call: the NSC partial sums meet by shuffle) into sc[] and the running max
    __device__ __forceinline__ void score_pos(int p, const KeyBlock& k, int n_ctx, float& lmax) const {
        float s = 0.f;
        if (p < n_ctx) s = p >= seqlen ? score_new(p - seqlen) : score_blk(k);
#pragma unroll
        for (int o = 1; o < TPR; o <<= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (p < n_ctx) {
            if (kblk == 0) sc[p - p_lo] = s;
            lmax = fmaxf(lmax, s);
        }
    }

    // scores of positions [p_lo, n_ctx): the staged window, then the ring, then (rows appended by this step, and without the
    // ring everything beyond the window) the cache.  Returns this thread's max.
    __device__ __forceinline__ float scores(int n_ctx) const {
        float lmax = -INFINITY;
        const int st_end = p_lo + n_st;                      // positions below are in shared memory
        int pb = p_lo;
        for (; pb < n_ctx && pb < st_end; pb += RPP) {
            const int pp = pb + krow;
            KeyBlock k = key_none();
            if (pp < st_end) k = key_block<false>(kst + (pp - p_lo) * ROWBK, ksst + (pp - p_lo) * NSC);
            else if (pp < min(n_ctx, seqlen)) k = key_global(pp);
            score_pos(pp, k, n_ctx, lmax);
        }
        if (ntail > 0) {
            ring_pass<ROWBK>(P.k_q, P.k_s, [&](int base, const uint8_t* rq_t, const half* rs_t) {
#pragma unroll 1
                for (int r0 = 0; r0 < SUB; r0 += RPP) {
                    if (base + r0 >= n_ctx) break;
                    const int rr = r0 + krow, pp = base + rr;
                    // an 8-bit sub-chunk can hold fewer positions than one pass scores (hd 64: 64 < RPP = 128): rows past
                    // the sub-chunk belong to the next one and are neither read nor scored here
                    const bool in_sub = SUB >= RPP || rr < SUB;
                    KeyBlock k = key_none();
                    if (in_sub && pp < c_hi) k = key_block<false>(rq_t + rr * ROWB, rs_t + rr * NSC);
                    score_pos(in_sub ? pp : INT_MAX, k, n_ctx, lmax);
                }
            });
            pb = p_lo + n_st + ntail * SUB;
        }
        constexpr int TU = 2 / KW;                           // rows per thread in flight: 32 bytes of keys in every format
        for (; pb < n_ctx; pb += TU * RPP) {
            KeyBlock k[TU];
#pragma unroll
            for (int u = 0; u < TU; ++u) {
                const int pp = pb + u * RPP + krow;
                k[u] = key_none();
                if (pp < min(n_ctx, seqlen)) k[u] = key_global(pp);
            }
#pragma unroll
            for (int u = 0; u < TU; ++u)
                if (pb + u * RPP < n_ctx) score_pos(pb + u * RPP + krow, k[u], n_ctx, lmax);
        }
        return lmax;
    }

    // ---- softmax over the CTA's positions: max and sum (mx, denom), sc[] becomes exp2(score - mx)
    __device__ __forceinline__ void softmax(float lmax, int n_ctx, float& mx, float& denom) const {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
        if (lane == 0) wred[warp] = lmax;
        __syncthreads();
        EXL2B_STAMP(P, 4);
        mx = wred[0];
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
        denom = 0.f;
#pragma unroll
        for (int w = 0; w < AQ_WARPS; ++w) denom += wred[AQ_WARPS + w];
    }

    // ---- P V in the rotated domain: lane = VEC consecutive values, warps stride over positions
    struct ValueRow {
        uint32_t x;       // 4 bits: the lane's nibbles | fp16 scale << 16;  8 bits: the fp16 scale
        uint32_t d;       // 8 bits: the lane's VEC bytes
    };
    __device__ __forceinline__ static ValueRow value_none() {
        if constexpr (VB == 4) return {0x8888u, 0u};
        else return {0u, 0x80808080u};
    }
    // this lane's values of a cached value row and their scale: in shared memory (staged window, ring), or (GLOBAL) in the cache
    template <bool GLOBAL>
    __device__ __forceinline__ ValueRow value_row(const uint8_t* rowq, const half* rows) const {
        const uint32_t s = ld_rows<GLOBAL>(reinterpret_cast<const uint16_t*>(rows) + ((lane * VEC) >> 5));
        if constexpr (VB == 4) {
            uint32_t x;
            if constexpr (VEC == 4) x = ld_rows<GLOBAL>(reinterpret_cast<const uint16_t*>(rowq) + lane);
            else x = (uint32_t)ld_rows<GLOBAL>(rowq + lane) | 0x8800u;
            return {x | (s << 16), 0u};
        } else {
            if constexpr (VEC == 4) return {s, ld_rows<GLOBAL>(reinterpret_cast<const uint32_t*>(rowq) + lane)};
            else return {s, (uint32_t)ld_rows<GLOBAL>(reinterpret_cast<const uint16_t*>(rowq) + lane)};
        }
    }
    __device__ __forceinline__ void pv_fma(float (&acc)[VEC], const ValueRow& v, float pw) const {
        if constexpr (VB == 4) {
            const float pe = pw * __half2float(__ushort_as_half((unsigned short)(v.x >> 16)));
#pragma unroll
            for (int j = 0; j < VEC; ++j) acc[j] = fmaf(pe, nib_f((v.x >> (4 * j)) & 15u), acc[j]);
        } else {
            const float pe = pw * __half2float(__ushort_as_half((unsigned short)v.x));
#pragma unroll
            for (int j = 0; j < VEC; ++j) acc[j] = fmaf(pe, byte_f((v.d >> (8 * j)) & 0xffu), acc[j]);
        }
    }

    // sum_p sc[p] v_p over [p_lo, n_ctx), per warp into red[warp]: the staged window, the ring, the cache, the new rows
    __device__ __forceinline__ void pv(int n_ctx) const {
        float acc[VEC];
#pragma unroll
        for (int j = 0; j < VEC; ++j) acc[j] = 0.f;
        const int st_end = p_lo + n_st;
#pragma unroll 4
        for (int p = p_lo + warp; p < st_end; p += AQ_WARPS) {
            const int r = p - p_lo;
            pv_fma(acc, value_row<false>(vst + r * ROWBV, vsst + r * NSC), sc[r]);
        }
        if (ntail > 0) {
            ring_pass<ROWBV>(P.v_q, P.v_s, [&](int base, const uint8_t* rq_t, const half* rs_t) {
#pragma unroll 4
                for (int r = warp; r < SUB; r += AQ_WARPS) {
                    const int pp = base + r;
                    if (pp < c_hi) pv_fma(acc, value_row<false>(rq_t + r * ROWB, rs_t + r * NSC), sc[pp - p_lo]);
                }
            });
        }
        for (int p0 = (ntail > 0 ? c_hi : st_end) + warp; p0 < c_hi; p0 += AQ_WARPS * 8) {   // without the ring: 8 rows in flight from global
            ValueRow v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int p = p0 + u * AQ_WARPS;
                v[u] = value_none();
                if (p < c_hi) {
                    const size_t r = row(p);
                    v[u] = value_row<true>(P.v_q + r * ROWBV, P.v_s + r * NSC);
                }
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int p = p0 + u * AQ_WARPS;
                if (p < c_hi) pv_fma(acc, v[u], sc[p - p_lo]);
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
    }

    // ---- single query, every cached row of the CTA in the staged window (CTA-uniform): staged_pass instead of scores /
    //      softmax / pv
    __device__ __forceinline__ bool all_staged() const { return P.q_len == 1 && ntail == 0 && c_hi - p_lo <= n_st; }
    // Each warp attends a contiguous range of the CTA's positions [p_lo, p_hi) (the appended row included, where it falls) on
    // its own: G positions per step scored as in scores() (TPR lanes each), a running max m and sum l, P V accumulated in
    // pv()'s layout with each weight shuffled from its position's lanes -- no score buffer, no barrier.  One barrier, then the
    // warps' (m, l, output) merge in warp order with weights exp2(m_w - M), end_query's split-KV merge, into (M, L, w) on
    // warps < UNITS (the triple end_query takes).  Reads only shared memory and writes only red / wred: it may also run on
    // whatever shared memory holds, with its results discarded (attn_q4_kernel runs it once before the dependency wait).
    __device__ __forceinline__ void staged_pass(float& M, float& L, float2& w) const {
        constexpr int G = 32 / TPR;
        const int per = (p_hi - p_lo + AQ_WARPS * G - 1) / (AQ_WARPS * G) * G;      // whole steps per warp
        const int lo = p_lo + warp * per, hi = min(p_hi, lo + per), c_end = min(hi, seqlen);
        const float* y_new = new_y + AQ_MAX_QLEN * HD + lane * VEC;                 // the appended value row, this lane's part
        float m = -INFINITY, l = 0.f, acc[VEC];
#pragma unroll
        for (int j = 0; j < VEC; ++j) acc[j] = 0.f;
        for (int pb = lo; pb < hi; pb += G) {
            const int pp = pb + lane / TPR;
            float s = 0.f;
            if (pp < c_end) s = score_blk(key_block<false>(kst + (pp - p_lo) * ROWBK, ksst + (pp - p_lo) * NSC));
            else if (pp < hi) s = score_new(0);
#pragma unroll
            for (int o = 1; o < TPR; o <<= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (pp >= hi) s = -INFINITY;
            float mn = s;
#pragma unroll
            for (int o = TPR; o < 32; o <<= 1) mn = fmaxf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
            mn = fmaxf(m, mn);                                   // finite: position pb is in range
            const float a = exp2f(m - mn), e = exp2f(s - mn);
            m = mn;
            l = fmaf(l, a, kblk == 0 ? e : 0.f);                 // each position counted on its first lane
#pragma unroll
            for (int j = 0; j < VEC; ++j) acc[j] *= a;
#pragma unroll 2
            for (int r = 0; r < G; ++r) {
                const int p = pb + r;
                const float pw = __shfl_sync(0xffffffffu, e, r * TPR);
                if (p < c_end) {
                    pv_fma(acc, value_row<false>(vst + (p - p_lo) * ROWBV, vsst + (p - p_lo) * NSC), pw);
                } else if (p < hi) {
#pragma unroll
                    for (int j = 0; j < VEC; ++j) acc[j] = fmaf(pw, y_new[j], acc[j]);
                }
            }
        }
#pragma unroll
        for (int o = TPR; o < 32; o <<= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
#pragma unroll
        for (int j = 0; j < VEC; ++j) red[warp * HD + lane * VEC + j] = acc[j];
        if (lane == 0) {
            wred[warp] = m;
            wred[AQ_WARPS + warp] = l;
        }
        EXL2B_STAMP(P, 4);
        __syncthreads();
        EXL2B_STAMP(P, 5);
        M = -INFINITY;
        L = 0.f;
        w = make_float2(0.f, 0.f);
        if (warp < UNITS) {          // elements warp * 64 + 2 lane, +1 of the rotated output (a warp with no positions weighs 0)
#pragma unroll
            for (int ww = 0; ww < AQ_WARPS; ++ww) M = fmaxf(M, wred[ww]);
#pragma unroll
            for (int ww = 0; ww < AQ_WARPS; ++ww) {
                const float wgt = exp2f(wred[ww] - M);
                const float2 a = reinterpret_cast<const float2*>(red + ww * HD + warp * 64)[lane];
                w.x = fmaf(wgt, a.x, w.x);
                w.y = fmaf(wgt, a.y, w.y);
                L = fmaf(wgt, wred[AQ_WARPS + ww], L);
            }
        }
    }

    // ---- the rows appended by this step go to the cache, from shared memory, on one warp
    __device__ __forceinline__ void append() const {
        constexpr int WK = ROWBK / 4, WV = ROWBV / 4;                 // 32-bit words per key / value row
        for (int idx = lane; idx < P.q_len * (WK + WV); idx += 32) {
            const int kv = idx >= P.q_len * WK, r = kv ? idx - P.q_len * WK : idx;
            const int ii = kv ? r / WV : r / WK, wd = kv ? r - ii * WV : r - ii * WK;
            const size_t rw = row(seqlen + ii);
            reinterpret_cast<uint32_t*>(kv ? P.v_q + rw * ROWBV : P.k_q + rw * ROWBK)[wd] =
                reinterpret_cast<const uint32_t*>(new_q + (kv ? AQ_MAX_QLEN * ROWBK + ii * ROWBV : ii * ROWBK))[wd];
        }
        for (int idx = lane; idx < 2 * P.q_len * NSC; idx += 32) {
            const int kv = idx / (P.q_len * NSC), r = idx - kv * P.q_len * NSC;
            const int ii = r / NSC, sidx = r - ii * NSC;
            (kv ? P.v_s : P.k_s)[row(seqlen + ii) * NSC + sidx] = new_s[(kv * AQ_MAX_QLEN + ii) * NSC + sidx];
        }
    }

    // ---- end of query i: sum over warps, (merge the splits,) rotate back (x = H y / 32), normalise, store.
    //      False: this CTA is done (it left its split's partial result, or merged them all).
    // elements warp * 64 + 2 lane, +1 of the rotated output (warp < UNITS), summed over the warps' P V sums
    __device__ __forceinline__ float2 warp_sum() const {
        float2 w = make_float2(0.f, 0.f);
#pragma unroll
        for (int ww = 0; ww < AQ_WARPS; ++ww) {
            w.x += red[ww * HD + warp * 64 + 2 * lane];
            w.y += red[ww * HD + warp * 64 + 2 * lane + 1];
        }
        return w;
    }
    __device__ __forceinline__ void store_out(int i, float2 w, float L) const {
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
                P.out_xp[(size_t)(k0 >> 3) * (P.out_tw * 8) + m * 8 + (k0 & 7)] = __low2half(o2);
                P.out_xp[(size_t)(k1 >> 3) * (P.out_tw * 8) + m * 8 + (k1 & 7)] = __high2half(o2);
            }
        }
    }
    __device__ __forceinline__ bool end_query(int i, float mx, float denom) const {
        return end_query(i, mx, denom, [&] { return warp_sum(); });
    }
    // the same with the CTA's unnormalised rotated output from `out()` (warps < UNITS) instead of this query's P V sums
    template <typename F>
    __device__ __forceinline__ bool end_query(int i, float mx, float denom, F&& out) const {
        if (ns_act > 1) {
            __shared__ int s_last;
            // leave (unnormalised rotated output, max, sum) of this chunk; the last CTA of the (head, sequence) merges them all
            float* wsp = P.ws + (((size_t)b * P.H + h) * P.nsplit + z) * (HD + 2);
            if (warp < UNITS) __stcg(reinterpret_cast<float2*>(wsp + warp * 64) + lane, out());
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
            if (s_last && warp < UNITS) {
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
                store_out(i, w, L);
            }
            return false;
        }
        if (warp < UNITS) store_out(i, out(), denom);
        if (i + 1 < P.q_len) __syncthreads();      // the next query reuses the shared buffers; after the last, the CTA leaves
        return true;
    }
};

template <int HD, int KB, int VB>
__global__ void __launch_bounds__(AQ_THREADS, 2) attn_q4_kernel(const __grid_constant__ AttnQ4Params P) {
    extern __shared__ __align__(16) uint8_t smem[];
    EXL2B_STAMP(P, 0);
    griddep_launch_dependents();
    if ((int)blockIdx.x >= P.busy_ctas) {          // slot holder: keeps this SM's slot until the working CTAs are done
        if (threadIdx.x == 0) slot_hold(P.slot_cnt, P.busy_ctas);
        return;
    }
    AttnCta<HD, KB, VB> c(P, smem);
    // the first cached K row of every thread and the first 16 cached V rows of every warp are already in shared memory when
    // q / k_new / v_new arrive
    if (!c.prologue()) return cta_exit(P);
    EXL2B_STAMP(P, 1);
    const auto after_wait = [&] {
        c.load_static();
        griddep_wait();
        EXL2B_STAMP(P, 2);
        c.new_rows_and_first_query();
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();
        EXL2B_STAMP(P, 3);
        EXL2B_STAMP(P, 8);
    };
    if (c.all_staged()) {
        // The warp-local pass (staged_pass) runs twice from ONE copy of its code: first before the dependency wait, on whatever
        // shared memory holds, its results discarded; then for real.  The first run costs nothing on the critical path (the
        // CTA waits for the Q|K|V launch anyway) and leaves the pass's instructions in this SM's instruction cache.  The
        // evict-first policy of the weight and cache streams (common.cuh) does not make this run redundant: without it the
        // pass takes ~4.4 us after the wait, with it ~2.6 us (DESIGN §7).
        float M = 0.f, L = 0.f;
        float2 w = make_float2(0.f, 0.f);
#pragma unroll 1
        for (int round = HD == 128 ? 0 : 1; round < 2; ++round) {      // (at HD 64 the first run spills: not done)
            if (round == 1) after_wait();
            c.staged_pass(M, L, w);
        }
        if (P.dbg && threadIdx.x == 0) atomicAdd(P.dbg + 10, 1ull);
        // the last warp appends (it has no part in the end of the query): nothing on the way to the output waits for these stores
        if (c.warp == AQ_WARPS - 1 && c.h % c.group == 0 && c.z == 0) c.append();
        if (!c.end_query(0, M, L, [&] { return w; })) return cta_exit(P);
    } else {
        after_wait();
        for (int i = 0; i < P.q_len; ++i) {
            const int n_ctx = (P.nsplit > 1) ? c.p_hi : c.seqlen + i + 1;          // end of the positions this CTA attends for query i
            if (i > 0) {                         // (the first query was rotated above, next to the quantisation)
                if (c.warp < c.UNITS) c.rotate_q(i, c.warp);
                __syncthreads();
            }
            const float lmax = c.scores(n_ctx);
            EXL2B_STAMP(P, 9);
            float mx, denom;
            c.softmax(lmax, n_ctx, mx, denom);
            c.pv(n_ctx);
            __syncthreads();
            EXL2B_STAMP(P, 5);
            // the last warp appends (it has no part in the end of the query): nothing on the way to the output waits for these stores
            if (i == P.q_len - 1 && c.warp == AQ_WARPS - 1 && c.h % c.group == 0 && c.z == 0) c.append();
            if (!c.end_query(i, mx, denom)) return cta_exit(P);
        }
    }
    if (P.dbg && threadIdx.x == 0) atomicMax(P.dbg + 7, globaltimer());
    cta_exit(P);
}

// Single-token decode over a cache too long for attn_q4_kernel's score buffer (attn_launch_plan, pass_len): the same phases,
// run once per pass of at most P.pass_len positions over the CTA's share [p_lo, p_hi) (the whole context, or one split-KV
// chunk).  Each pass scores, exponentiates against its own max and sums its P V; the CTA carries a running max M, sum L and
// rotated output across passes, rescaled by exp2(M_old - M_new) -- end_query's split-KV merge, done in sequence -- and hands
// the final (M, L, output) to end_query.  The staged window belongs to the first pass; every later cached row streams through
// the ring.  The appended row (position seqlen) is in the last pass of the last chunk.
template <int HD, int KB, int VB>
__global__ void __launch_bounds__(AQ_THREADS, 2) attn_q4_passes_kernel(const __grid_constant__ AttnQ4Params P) {
    extern __shared__ __align__(16) uint8_t smem[];
    EXL2B_STAMP(P, 0);
    griddep_launch_dependents();
    if ((int)blockIdx.x >= P.busy_ctas) {
        if (threadIdx.x == 0) slot_hold(P.slot_cnt, P.busy_ctas);
        return;
    }
    AttnCta<HD, KB, VB> c(P, smem);
    if (!c.prologue()) return cta_exit(P);
    EXL2B_STAMP(P, 1);
    c.load_static();
    griddep_wait();
    EXL2B_STAMP(P, 2);
    c.new_rows_and_first_query();
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    EXL2B_STAMP(P, 3);
    // the running output, elements warp * 64 + 2 lane, +1 on warps < UNITS, each read and written by its own thread only.  It
    // lives in new_y's second key row, which a single query leaves unused (registers would spill at Q4 hd 128).
    float2* o = reinterpret_cast<float2*>(c.new_y + HD) + c.warp * 32 + c.lane;
    if (c.warp < c.UNITS) *o = make_float2(0.f, 0.f);
    float M = -INFINITY, L = 0.f;
    for (int pl = c.p_lo, nst = c.n_st; pl < c.p_hi; pl += P.pass_len, nst = 0) {
        const int ph = min(c.p_hi, pl + P.pass_len);
        c.begin_pass(pl, ph, nst);
        const float lmax = c.scores(ph);
        float mx, denom;
        c.softmax(lmax, ph, mx, denom);
        c.pv(ph);
        __syncthreads();
        const float mn = fmaxf(M, mx), a = exp2f(M - mn), w = exp2f(mx - mn);
        if (c.warp < c.UNITS) {
            const float2 s = c.warp_sum(), r = *o;
            *o = make_float2(fmaf(w, s.x, r.x * a), fmaf(w, s.y, r.y * a));
        }
        L = fmaf(w, denom, L * a);
        M = mn;
    }
    EXL2B_STAMP(P, 5);
    if (c.warp == AQ_WARPS - 1 && c.h % c.group == 0 && c.z == 0) c.append();
    if (!c.end_query(0, M, L, [&] { return *o; })) return cta_exit(P);
    if (P.dbg && threadIdx.x == 0) atomicMax(P.dbg + 7, globaltimer());
    cta_exit(P);
}

// The launch of one call, from the shape and the SM count alone (tests/attn_regimes.py restates it)
struct AttnLaunch {
    int nsplit;          // CTAs per (head, sequence)
    int sc_len;          // floats of the score buffer
    int ring_slots;      // AQ_RING with the ring, else 0
    int stage;           // staged cached positions per CTA
    int pass_len;        // > 0: attn_q4_passes_kernel with passes of this many positions (= sc_len); 0: attn_q4_kernel
    AttnSmem smem;
};
static AttnLaunch attn_launch_plan(int kb, int vb, int hd, int q_len, int num_heads, int batch, int page_size, int pages_per_seq,
                                   int sms) {
    AttnLaunch L;
    const int max_ctx = page_size * pages_per_seq;
    // split-KV: only for single-query decode over caches long enough to need it
    L.nsplit = 1;
    if (q_len == 1 && max_ctx > 2 * AQ_SPLIT_MIN) {
        const int by_ctx = (max_ctx + AQ_SPLIT_MIN - 1) / AQ_SPLIT_MIN;
        const int by_sms = std::max(1, (2 * sms) / std::max(1, num_heads * batch));
        L.nsplit = std::max(1, std::min(std::min(by_ctx, by_sms), 16));
    }
    L.sc_len = L.nsplit > 1 ? std::max(AQ_SPLIT_MIN, (max_ctx + L.nsplit) / L.nsplit) + 8 : max_ctx + q_len;
    // cached rows beyond the staged window: streamed through a ring of 4 sub-chunks (128 positions at Q4) when the cache is long;
    // the ring takes the place of half the staged window, so the CTA keeps the footprint that lets it share an SM with one GEMV
    // CTA (a first version that ADDED the ring lost that co-residency).  The ring pays once a CTA has thousands of positions;
    // below, the larger window wins.  The host only knows the cache's capacity:
    L.ring_slots = (max_ctx > 8192) ? AQ_RING : 0;
    // The window and the ring are sized in BYTES: every format stages at most the bytes of Q4's AQ_STAGE (or AQ_STAGE / 2 with
    // the ring) positions, in whole multiples of 64 positions, so no format needs more shared memory than Q4: Q8 stages 256
    // (128) positions, Q6 320 (128).  Ring sub-chunks hold the bytes of 128 Q4 rows of the wider of K and V (64 at 8 bits).
    const int rowk = hd * kb / 8, rowv = hd * vb / 8, nsc = hd / 32;
    const int window = L.ring_slots ? AQ_STAGE / 2 : AQ_STAGE;
    L.stage = (int)((size_t)window * (hd + 4 * nsc) / (size_t)(rowk + rowv + 4 * nsc)) / 64 * 64;
    L.smem = attn_smem_map(hd, kb, vb, pages_per_seq, L.sc_len, L.stage, L.ring_slots != 0);
    // A single query whose score buffer does not fit walks its positions in passes instead.  Its buffer then holds one pass,
    // as long as keeps the CTA within AQ_PASS_SMEM, in multiples of AQ_PASS_ALIGN, at least AQ_PASS_MIN.  (The ring is on: a score buffer of
    // ~29 000 positions or more means a cache far above 8192.)  Launches that fit keep the plan above.
    L.pass_len = 0;
    if (q_len == 1 && L.smem.total > (uint32_t)AQ_SMEM_MAX) {
        const uint32_t rest = attn_smem_map(hd, kb, vb, pages_per_seq, 0, L.stage, true).total;
        const int room = rest < (uint32_t)AQ_PASS_SMEM ? (int)((AQ_PASS_SMEM - rest) / 4) : 0;
        L.pass_len = std::max(AQ_PASS_MIN, room / AQ_PASS_ALIGN * AQ_PASS_ALIGN);
        L.sc_len = L.pass_len;
        L.smem = attn_smem_map(hd, kb, vb, pages_per_seq, L.sc_len, L.stage, true);
    }
    return L;
}

}  // namespace exl2b

using namespace exl2b;

static int32_t* g_attn_err[64] = {nullptr};

// the sticky status word of `device` that every fused attention kernel sets (exl2b_paged_attn_status), created on first use
namespace exl2b {
int attn_err_flag(int device, int32_t** flag) {
    if (!g_attn_err[device]) {
        EXL2B_CUDA(cudaMalloc(&g_attn_err[device], sizeof(int32_t)));
        EXL2B_CUDA(cudaMemset(g_attn_err[device], 0, sizeof(int32_t)));
    }
    *flag = g_attn_err[device];
    return 0;
}
}  // namespace exl2b

// Split-KV partial results and arrival counters, one set per (device, stream) like the wgmma workspace (gemv.cu): launches on
// different streams never merge each other's partials.  Allocated once at the bound every split launch fits in and never
// freed or moved, because a captured graph keeps the pointers it was captured with.  attn_launch_plan splits only when
// H * B <= SMs (by_sms >= 2) and takes nsplit <= 2 * SMs / (H * B), so B * H * nsplit <= 2 * SMs: at most 2 * SMs * (128 + 2)
// floats and SMs counters (tests/test_scratch_bound.py).  Created on first use: never inside a stream capture.
struct AttnScratch {
    float* ws = nullptr;
    unsigned int* cnt = nullptr;
    size_t ws_floats = 0, n_cnt = 0;
};
static std::map<std::pair<int, cudaStream_t>, AttnScratch> g_attn_scratch;
static std::mutex g_attn_scratch_mutex;

static int attn_scratch(int device, cudaStream_t stream, int sms, AttnScratch** out) {
    std::lock_guard<std::mutex> lock(g_attn_scratch_mutex);
    AttnScratch& s = g_attn_scratch[{device, stream}];
    if (!s.ws) {
        const size_t floats = (size_t)2 * sms * (128 + 2), cnt = (size_t)sms;
        EXL2B_CUDA(cudaMalloc(&s.ws, floats * sizeof(float)));
        EXL2B_CUDA(cudaMalloc(&s.cnt, cnt * sizeof(unsigned int)));
        EXL2B_CUDA(cudaMemset(s.cnt, 0, cnt * sizeof(unsigned int)));
        EXL2B_CUDA(cudaDeviceSynchronize());
        s.ws_floats = floats;
        s.n_cnt = cnt;
    }
    *out = &s;
    return 0;
}

// exl2b_debug_scratch, attention kinds: the workspace or counters of (device, stream), NULL / 0 before their first use
namespace exl2b {
int attn_scratch_query(int device, cudaStream_t stream, int kind, void** ptr, size_t* bytes) {
    std::lock_guard<std::mutex> lock(g_attn_scratch_mutex);
    const auto it = g_attn_scratch.find({device, stream});
    *ptr = nullptr;
    *bytes = 0;
    if (it == g_attn_scratch.end()) return 0;
    if (kind == EXL2B_SCRATCH_ATTN_WS) {
        *ptr = it->second.ws;
        *bytes = it->second.ws_floats * sizeof(float);
    } else {
        *ptr = it->second.cnt;
        *bytes = it->second.n_cnt * sizeof(unsigned int);
    }
    return 0;
}
}  // namespace exl2b

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

template <int KB, int VB>
static int attn_q_launch(int head_dim, dim3 grid, size_t smem, cudaStream_t stream, const AttnQ4Params& P) {
    if (P.pass_len) {
        if (head_dim == 128)
            EXL2B_CUDA(launch_pdl_f("attn", attn_q4_passes_kernel<128, KB, VB>, grid, dim3(AQ_THREADS), smem, stream, P));
        else
            EXL2B_CUDA(launch_pdl_f("attn", attn_q4_passes_kernel<64, KB, VB>, grid, dim3(AQ_THREADS), smem, stream, P));
        return 0;
    }
    if (head_dim == 128)
        EXL2B_CUDA(launch_pdl_f("attn", attn_q4_kernel<128, KB, VB>, grid, dim3(AQ_THREADS), smem, stream, P));
    else
        EXL2B_CUDA(launch_pdl_f("attn", attn_q4_kernel<64, KB, VB>, grid, dim3(AQ_THREADS), smem, stream, P));
    return 0;
}

template <int KB, int VB>
static int attn_q_set_smem() {
    EXL2B_CUDA(cudaFuncSetAttribute(attn_q4_kernel<128, KB, VB>, cudaFuncAttributeMaxDynamicSharedMemorySize, AQ_SMEM_MAX));
    EXL2B_CUDA(cudaFuncSetAttribute(attn_q4_kernel<64, KB, VB>, cudaFuncAttributeMaxDynamicSharedMemorySize, AQ_SMEM_MAX));
    EXL2B_CUDA(cudaFuncSetAttribute(attn_q4_passes_kernel<128, KB, VB>, cudaFuncAttributeMaxDynamicSharedMemorySize, AQ_SMEM_MAX));
    EXL2B_CUDA(cudaFuncSetAttribute(attn_q4_passes_kernel<64, KB, VB>, cudaFuncAttributeMaxDynamicSharedMemorySize, AQ_SMEM_MAX));
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
        const int rows = batch * q_len;
        EXL2B_REQUIRE(rows <= GEMV_MAX_CHAIN_ROWS, "chained attention output needs at most %d rows (rows %d)", GEMV_MAX_CHAIN_ROWS, rows);
        const bool wide = rows > GEMV_MTOK;      // o_proj's launch runs on a wide tile and reads its 64-row buffer
        int rc = qmatrix_chain_buffers(oc, wide);
        if (rc) return rc;
        P.out_xp = wide ? oc->xp_wide : oc->xp_buf;
        P.out_invperm = oc->invperm;
        P.out_plain = (rows == 1 && gemv_i8_enabled()) ? 1 : 0;      // the single-row GEMV reads a plain fp16 row
        P.out_tw = tc_tile(rows);
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
    EXL2B_REQUIRE(dev >= 0 && dev < 64, "bad device");
    const int sms = device_sm_count(dev);
    const AttnLaunch L = attn_launch_plan(kb, vb, head_dim, q_len, num_heads, batch, page_size, pages_per_seq, sms);
    if (L.pass_len)
        EXL2B_REQUIRE(L.smem.total <= AQ_SMEM_MAX,
                      "a page table of %d pages needs %u bytes of shared memory with passes of %d positions, above %d",
                      pages_per_seq, L.smem.total, L.pass_len, AQ_SMEM_MAX);
    EXL2B_REQUIRE(L.smem.total <= AQ_SMEM_MAX, "context of %d tokens does not fit the score buffer", P.max_ctx);
    {
        int rc = attn_err_flag(dev, &P.err);
        if (rc) return rc;
    }
    if (L.nsplit > 1) {
        AttnScratch* s = nullptr;
        int rc = attn_scratch(dev, (cudaStream_t)stream, sms, &s);
        if (rc) return rc;
        const size_t need = (size_t)batch * num_heads * L.nsplit * (head_dim + 2), need_c = (size_t)batch * num_heads;
        EXL2B_REQUIRE(need <= s->ws_floats && need_c <= s->n_cnt,
                      "split-KV launch needs %zu floats / %zu counters, above the per-stream bound %zu / %zu", need, need_c,
                      s->ws_floats, s->n_cnt);
        P.ws = s->ws;
        P.cnt = s->cnt;
    }
    P.nsplit = L.nsplit;
    P.sc_len = L.sc_len;
    P.ring_slots = L.ring_slots;
    P.stage = L.stage;
    P.pass_len = L.pass_len;
    P.dbg = exl2b::g_dbg ? exl2b::g_dbg + 32 * (exl2b::g_dbg_slot++ % 64) : nullptr;
    P.dbg_cta = 0;
    static bool attr_set[64] = {false};
    if (!attr_set[dev]) {
        int rc = attn_q_set_smem<4, 4>();
        if (!rc) rc = attn_q_set_smem<8, 4>();
        if (!rc) rc = attn_q_set_smem<8, 8>();
        if (rc) return rc;
        attr_set[dev] = true;
    }
    static SlotCounters slot_cnts;
    int rc = next_slot_counter(slot_cnts, dev, &P.slot_cnt);
    if (rc) return rc;
    P.batch = batch;
    P.busy_ctas = num_heads * batch * L.nsplit;
    dim3 grid(slot_holders_disabled() ? P.busy_ctas : std::max(P.busy_ctas, sms));
    if (wbits == 4) return attn_q_launch<4, 4>(head_dim, grid, L.smem.total, (cudaStream_t)stream, P);
    if (wbits == 6) return attn_q_launch<8, 4>(head_dim, grid, L.smem.total, (cudaStream_t)stream, P);
    return attn_q_launch<8, 8>(head_dim, grid, L.smem.total, (cudaStream_t)stream, P);
}
