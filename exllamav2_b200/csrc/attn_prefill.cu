// Prompt attention straight over the Q4 / Q6 / Q8 K/V cache: attend, quantise and append the new rows, in ONE kernel, for any
// number of new rows per sequence (the decode kernel, attn_q4.cu, takes at most 8).
//
// The reference runs, per layer and prompt chunk (exllamav2/attn.py:560-621, cache.py:472-556):
//     q_to_fp16_kv over the WHOLE live cache -> flash_attn_with_kvcache on the fp16 temp -> fp16_to_q_kv of the new rows.
// Here the cache is read as stored and the scores and P V products run on tensor cores (mma.sync.m16n8k16, fp16 operands,
// fp32 accumulation), flash-attention style: an online softmax over tiles of AP_BN key positions.
//   * Rotated domain, as in the decode kernel: the cache holds y = H32 x per 64-value unit (kv_format.cuh), H symmetric with
//     H H = 32 I, so q . x = (H q) . y / 32 and sum_s p_s x_s = H (sum_s p_s y_s) / 32.  The query tile is rotated once in fp32
//     with softmax_scale * log2(e) / 32 folded in, then rounded to fp16; the output tile is rotated back once, in fp32.
//   * Cached rows are dequantised to half(code - Z) * scale in fp16 -- the first step of the reference's unpack, bit for bit --
//     with no per-position butterfly.
//   * The q_len new rows are attended UNQUANTISED, as in the reference, where flash-attn sees the fp16 rows and the cache
//     quantises them afterwards: rotated by the fp32 butterfly (hadamard32_f) and rounded to fp16.
//   * GQA: the M dimension of a CTA's tile is (token, head in group) pairs of one kv head, so every dequantised K / V tile
//     serves all the query heads that read it.  Any ratio H / KVH works (7 included).
//   * The new rows are quantised with the cache's own arithmetic (kv_format.cuh, as kvcache.cu pack_unit) and written at
//     [seqlen, seqlen + q_len): each new 64-value unit by exactly one CTA, and only the new tokens' units.
// Why mma.sync and not wgmma: every operand tile is produced in shared memory by this CTA's own threads (dequantised keys,
// transposed values, rotated queries) and the P operand comes straight from the score accumulators in registers, which is the
// m16n8k16 fragment layout; a 64-row tile of 4 warps keeps two CTAs per SM with no warpgroup-wide synchronisation.
#include "kv_format.cuh"

namespace exl2b {

int attn_err_flag(int device, int32_t** flag);      // attn_q4.cu

constexpr int AP_THREADS = 128;
constexpr int AP_WARPS = 4;
constexpr int AP_BM = 64;                  // (token, head in group) rows per CTA: 16 per warp
constexpr int AP_BN = 64;                  // key positions per tile (a page holds whole tiles: page_size % AP_BN == 0)
constexpr int AP_SMEM_MAX = 200 * 1024;    // dynamic shared memory a launch may use

// dynamic shared-memory map of a CTA (byte offsets) -- one definition for the kernel and the host that sizes the launch
struct PrefillSmem {
    uint32_t q, kh, vt, out, raw, stage, pages, total;
};
__host__ __device__ inline PrefillSmem prefill_smem_map(int hd, int kb, int vb, int pages_per_seq) {
    const uint32_t nsc = hd / 32, rowk = hd * kb / 8, rowv = hd * vb / 8;
    PrefillSmem m;
    m.q = 0;                                            // [AP_BM][hd + 8]  rotated, scaled queries, fp16
    m.kh = m.q + AP_BM * (hd + 8) * 2;                  // [AP_BN][hd + 8]  the tile's keys, fp16 (rotated domain)
    m.vt = m.kh + AP_BN * (hd + 8) * 2;                 // [hd][AP_BN + 8]  the tile's values, fp16, transposed
    m.out = 0;                                          // [AP_BM][hd + 4]  output tile, fp32: over q / kh / vt once they are done
    const uint32_t tiles = m.vt + hd * (AP_BN + 8) * 2, out_end = AP_BM * (hd + 4) * 4;
    m.raw = tiles > out_end ? tiles : out_end;          // [2] stages of cp.async bytes: K codes, V codes, K scales, V scales
    m.stage = AP_BN * (rowk + rowv + 2 * nsc * 2);
    m.pages = m.raw + 2 * m.stage;                      // [pages_per_seq]  the sequence's page table
    m.total = m.pages + ((pages_per_seq + 3) & ~3) * 4;
    return m;
}

struct PrefillParams {
    const half* q;                  // [batch, q_len, H, hd]     (RoPE already applied)
    const half* k_new;              // [batch, q_len, KVH, hd]
    const half* v_new;
    uint8_t* k_q;                   // [pages, page_size, KVH, hd * KB / 8]
    half* k_s;                      // [pages, page_size, KVH, hd / 32]
    uint8_t* v_q;
    half* v_s;
    const int32_t* cache_seqlens;   // [batch]
    const int32_t* block_table;     // [batch, pages_per_seq]
    half* out;                      // [batch, q_len, H, hd]
    int q_len, H, KVH, group, page_size, pages_per_seq, max_ctx;
    float scale_log2;               // softmax_scale * log2(e)
    int32_t* err;                   // sticky status: bit 0 = a sequence ran past its page table (nothing appended, no output)
};

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    const half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}

// Grid (ceil(q_len * group / AP_BM), KVH, batch).  CTA (mb, kvh, b) owns rows [mb * AP_BM, +AP_BM) of the pairs r = t * group + j
// (token t, query head kvh * group + j) of sequence b.  Query t sees positions [0, seqlen + t].
//
// Invariant that keeps the append race-free: positions >= seqlen are read ONLY from k_new / v_new, never from the cache, by
// every CTA; the cache is written only at positions >= seqlen.  So no CTA can read a unit another CTA is appending.
template <int HD, int KB, int VB>
__global__ void __launch_bounds__(AP_THREADS, 2) attn_prefill_kernel(const __grid_constant__ PrefillParams P) {
    static_assert(HD == 64 || HD == 128, "head_dim 64 or 128");
    constexpr int ROWBK = HD * KB / 8, ROWBV = HD * VB / 8, NSC = HD / 32, UNITS = HD / 64;
    constexpr int QP = HD + 8, VP = AP_BN + 8, OP = HD + 4;       // row pitches (halves, halves, floats): conflict-free fragments
    constexpr int KS = HD / 16, NT = AP_BN / 8, DT = HD / 8;      // k-steps of Q K^T, key n-tiles, output n-tiles
    extern __shared__ __align__(16) uint8_t smem[];
    const PrefillSmem m = prefill_smem_map(HD, KB, VB, P.pages_per_seq);
    half* qs = reinterpret_cast<half*>(smem + m.q);
    half* kh = reinterpret_cast<half*>(smem + m.kh);
    half* vt = reinterpret_cast<half*>(smem + m.vt);
    float* os = reinterpret_cast<float*>(smem + m.out);
    int* pages = reinterpret_cast<int*>(smem + m.pages);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, gq = lane >> 2, tig = lane & 3;
    const int kvh = blockIdx.y, b = blockIdx.z, g = P.group;
    const int rows = P.q_len * g, m0 = blockIdx.x * AP_BM;

    griddep_wait();
    const int seqlen = P.cache_seqlens[b];
    if (seqlen < 0 || seqlen + P.q_len > P.max_ctx) {          // the page table ends here: refuse instead of corrupting
        if (tid == 0) atomicOr(P.err, 1);
        return;
    }
    const int t_hi = min(P.q_len - 1, (min(m0 + AP_BM, rows) - 1) / g);     // last token of the CTA
    const int n_end = seqlen + t_hi + 1;                                       // positions it attends: [0, n_end)
    const int32_t* bt = P.block_table + (size_t)b * P.pages_per_seq;
    for (int i = tid; i < (seqlen + P.q_len + P.page_size - 1) / P.page_size; i += AP_THREADS) pages[i] = bt[i];
    __syncthreads();
    auto cache_row = [&](int p) -> size_t { return ((size_t)pages[p / P.page_size] * P.page_size + p % P.page_size) * P.KVH + kvh; };

    // ---- cp.async of the cached bytes of key tile j into stage j & 1 (one commit group per call, possibly empty)
    auto issue = [&](int j) {
        uint8_t* kr = smem + m.raw + (j & 1) * m.stage;
        uint8_t* vr = kr + AP_BN * ROWBK;
        half* ksr = reinterpret_cast<half*>(vr + AP_BN * ROWBV);
        half* vsr = ksr + AP_BN * NSC;
        const int p0 = j * AP_BN, nc = min(AP_BN, seqlen - p0);
        if (nc > 0) {
            const size_t r0 = cache_row(p0);               // a tile lies in one page: its rows are KVH rows apart
            constexpr int CHK = ROWBK / 16, CH = CHK + ROWBV / 16;
            for (int idx = tid; idx < nc * CH; idx += AP_THREADS) {
                const int pos = idx / CH, ch = idx - pos * CH;
                const size_t r = r0 + (size_t)pos * P.KVH;
                if (ch < CHK) cp_async16(smem_addr(kr + pos * ROWBK + ch * 16), P.k_q + r * ROWBK + ch * 16);
                else cp_async16(smem_addr(vr + pos * ROWBV + (ch - CHK) * 16), P.v_q + r * ROWBV + (ch - CHK) * 16);
            }
            for (int idx = tid; idx < 2 * nc; idx += AP_THREADS) {
                const int kv = idx >= nc, pos = kv ? idx - nc : idx;
                const size_t r = r0 + (size_t)pos * P.KVH;
                cp_async_small<NSC * 2>(smem_addr((kv ? vsr : ksr) + pos * NSC), (kv ? P.v_s : P.k_s) + r * NSC);
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    const int ntiles = (n_end + AP_BN - 1) / AP_BN;       // key tiles wholly beyond the CTA's last query are skipped
    issue(0);

    // ---- append: the new tokens t whose first row t * g lies in this CTA, quantised exactly as fp16_to_q_kv (pack_unit)
    {
        const int ta = (m0 + g - 1) / g, tb = min(P.q_len, (m0 + AP_BM + g - 1) / g);
        for (int job = warp; job < (tb - ta) * UNITS * 2; job += AP_WARPS) {
            const int kv = job & 1, r = job >> 1, un = r % UNITS, t = ta + r / UNITS;
            const half* src = (kv ? P.v_new : P.k_new) + (((size_t)b * P.q_len + t) * P.KVH + kvh) * HD + un * 64;
            const half2 w2 = hadamard32_h(reinterpret_cast<const half2*>(src)[lane], lane);
            const size_t row = cache_row(seqlen + t);
            half* sc = (kv ? P.v_s : P.k_s) + row * NSC + un * 2 + (lane >> 4);
            if ((kv ? VB : KB) == 4) {
                const KvCodes c = kv_quantise<4>(w2);
                (kv ? P.v_q + row * ROWBV : P.k_q + row * ROWBK)[un * 32 + lane] = (uint8_t)(c.q0 | (c.q1 << 4));
                if ((lane & 15) == 0) *sc = c.scale;
            } else {
                const KvCodes c = kv_quantise<8>(w2);
                reinterpret_cast<uint16_t*>((kv ? P.v_q + row * ROWBV : P.k_q + row * ROWBK) + un * 64)[lane] = (uint16_t)(c.q0 | (c.q1 << 8));
                if ((lane & 15) == 0) *sc = c.scale;
            }
        }
    }

    // ---- query tile: H q * (softmax_scale * log2 e / 32) in fp32, rounded to fp16; rows past the last pair are zero
    const float fq = P.scale_log2 * (1.0f / 32.0f);
    for (int job = warp; job < AP_BM * UNITS; job += AP_WARPS) {
        const int r = job / UNITS, un = job - r * UNITS, R = m0 + r;
        float2 w = make_float2(0.f, 0.f);
        if (R < rows) {
            const int t = R / g, h = kvh * g + (R - t * g);
            const half* src = P.q + (((size_t)b * P.q_len + t) * P.H + h) * HD + un * 64;
            w = hadamard32_f(__half22float2(reinterpret_cast<const half2*>(src)[lane]), lane);
        }
        *reinterpret_cast<half2*>(qs + r * QP + un * 64 + 2 * lane) = __floats2half2_rn(w.x * fq, w.y * fq);
    }
    __syncthreads();
    const int r0 = warp * 16 + gq;                       // this thread's two rows of the warp's 16: r0, r0 + 8
    uint32_t qa[KS][4];
#pragma unroll
    for (int kk = 0; kk < KS; ++kk) {
        const half* a = qs + r0 * QP + kk * 16 + 2 * tig;
        qa[kk][0] = *reinterpret_cast<const uint32_t*>(a);
        qa[kk][1] = *reinterpret_cast<const uint32_t*>(a + 8 * QP);
        qa[kk][2] = *reinterpret_cast<const uint32_t*>(a + 8);
        qa[kk][3] = *reinterpret_cast<const uint32_t*>(a + 8 * QP + 8);
    }
    // last visible position of each of the two rows (rows past the last pair behave as the last token)
    const int lim0 = seqlen + min(P.q_len - 1, (m0 + r0) / g), lim1 = seqlen + min(P.q_len - 1, (m0 + r0 + 8) / g);
    float o[DT][4];
#pragma unroll
    for (int d = 0; d < DT; ++d) o[d][0] = o[d][1] = o[d][2] = o[d][3] = 0.f;
    float mx0 = -INFINITY, mx1 = -INFINITY, l0 = 0.f, l1 = 0.f;

    for (int j = 0; j < ntiles; ++j) {
        const int p0 = j * AP_BN;
        if (j + 1 < ntiles) issue(j + 1);
        else asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 1;" ::: "memory");
        __syncthreads();                                  // tile j's bytes are in; every warp is done with the last kh / vt
        // ---- dequantise the cached positions (one thread per 8 values of a K and a V row); zero the positions past n_end
        {
            const uint8_t* kr = smem + m.raw + (j & 1) * m.stage;
            const uint8_t* vr = kr + AP_BN * ROWBK;
            const half* ksr = reinterpret_cast<const half*>(vr + AP_BN * ROWBV);
            const half* vsr = ksr + AP_BN * NSC;
            const int nc = min(AP_BN, seqlen - p0), nv = min(AP_BN, n_end - p0);
            for (int idx = tid; idx < AP_BN * (HD / 8); idx += AP_THREADS) {
                const int pos = idx / (HD / 8), e0 = (idx - pos * (HD / 8)) * 8;
                if (pos >= nc && pos < nv) continue;      // a new row: below
                half2 kk[4], vv[4];
                if (pos < nc) {
                    int ck[8], cv[8];
                    if constexpr (KB == 4) {
                        const uint32_t w = *reinterpret_cast<const uint32_t*>(kr + pos * ROWBK + e0 / 2);
#pragma unroll
                        for (int i = 0; i < 8; ++i) ck[i] = (int)((w >> (4 * i)) & 15u) - 8;
                    } else {
                        const uint2 w = *reinterpret_cast<const uint2*>(kr + pos * ROWBK + e0);
#pragma unroll
                        for (int i = 0; i < 8; ++i) ck[i] = (int)(((i < 4 ? w.x : w.y) >> (8 * (i & 3))) & 255u) - 128;
                    }
                    if constexpr (VB == 4) {
                        const uint32_t w = *reinterpret_cast<const uint32_t*>(vr + pos * ROWBV + e0 / 2);
#pragma unroll
                        for (int i = 0; i < 8; ++i) cv[i] = (int)((w >> (4 * i)) & 15u) - 8;
                    } else {
                        const uint2 w = *reinterpret_cast<const uint2*>(vr + pos * ROWBV + e0);
#pragma unroll
                        for (int i = 0; i < 8; ++i) cv[i] = (int)(((i < 4 ? w.x : w.y) >> (8 * (i & 3))) & 255u) - 128;
                    }
                    const half2 sk = __half2half2(ksr[pos * NSC + e0 / 32]), sv = __half2half2(vsr[pos * NSC + e0 / 32]);
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        kk[i] = __hmul2(__halves2half2(__int2half_rn(ck[2 * i]), __int2half_rn(ck[2 * i + 1])), sk);
                        vv[i] = __hmul2(__halves2half2(__int2half_rn(cv[2 * i]), __int2half_rn(cv[2 * i + 1])), sv);
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < 4; ++i) kk[i] = vv[i] = __float2half2_rn(0.f);
                }
                *reinterpret_cast<uint4*>(kh + pos * QP + e0) = *reinterpret_cast<const uint4*>(kk);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    vt[(e0 + 2 * i) * VP + pos] = __low2half(vv[i]);
                    vt[(e0 + 2 * i + 1) * VP + pos] = __high2half(vv[i]);
                }
            }
            // ---- the new rows of the tile, from k_new / v_new (never from the cache): fp32 butterfly, rounded to fp16
            const int n_lo = max(0, seqlen - p0), jobs = max(0, nv - n_lo) * UNITS * 2;
            for (int job = warp; job < jobs; job += AP_WARPS) {
                const int kv = job & 1, r = job >> 1, un = r % UNITS, pos = n_lo + r / UNITS, t = p0 + pos - seqlen;
                const half* src = (kv ? P.v_new : P.k_new) + (((size_t)b * P.q_len + t) * P.KVH + kvh) * HD + un * 64;
                const float2 y = hadamard32_f(__half22float2(reinterpret_cast<const half2*>(src)[lane]), lane);
                const half2 yh = __floats2half2_rn(y.x, y.y);
                const int e = un * 64 + 2 * lane;
                if (!kv) {
                    *reinterpret_cast<half2*>(kh + pos * QP + e) = yh;
                } else {
                    vt[e * VP + pos] = __low2half(yh);
                    vt[(e + 1) * VP + pos] = __high2half(yh);
                }
            }
        }
        __syncthreads();
        // ---- S = Q~ K~^T on the warp's 16 rows, the tile's AP_BN keys
        float s[NT][4];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
            const half* bk = kh + (nt * 8 + gq) * QP + 2 * tig;
#pragma unroll
            for (int kk = 0; kk < KS; ++kk)
                mma16816(s[nt], qa[kk], *reinterpret_cast<const uint32_t*>(bk + kk * 16), *reinterpret_cast<const uint32_t*>(bk + kk * 16 + 8));
        }
        // causal mask where the tile reaches past a row's last visible position (the diagonal tiles, and the zeroed tail)
        if (p0 + AP_BN - 1 > min(lim0, lim1)) {
#pragma unroll
            for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const int p = p0 + nt * 8 + 2 * tig + (c & 1);
                    if (p > (c < 2 ? lim0 : lim1)) s[nt][c] = -INFINITY;
                }
        }
        // ---- online softmax (log2 domain); position 0 is visible to every row, so the running max is finite from tile 0 on
        float t0 = -INFINITY, t1 = -INFINITY;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            t0 = fmaxf(t0, fmaxf(s[nt][0], s[nt][1]));
            t1 = fmaxf(t1, fmaxf(s[nt][2], s[nt][3]));
        }
#pragma unroll
        for (int o2 = 1; o2 < 4; o2 <<= 1) {
            t0 = fmaxf(t0, __shfl_xor_sync(0xffffffffu, t0, o2));
            t1 = fmaxf(t1, __shfl_xor_sync(0xffffffffu, t1, o2));
        }
        const float n0 = fmaxf(mx0, t0), n1 = fmaxf(mx1, t1);
        const float c0 = exp2f(mx0 - n0), c1 = exp2f(mx1 - n1);
        mx0 = n0;
        mx1 = n1;
        l0 *= c0;
        l1 *= c1;
#pragma unroll
        for (int d = 0; d < DT; ++d) {
            o[d][0] *= c0;
            o[d][1] *= c0;
            o[d][2] *= c1;
            o[d][3] *= c1;
        }
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            s[nt][0] = exp2f(s[nt][0] - n0);
            s[nt][1] = exp2f(s[nt][1] - n0);
            s[nt][2] = exp2f(s[nt][2] - n1);
            s[nt][3] = exp2f(s[nt][3] - n1);
            l0 += s[nt][0] + s[nt][1];
            l1 += s[nt][2] + s[nt][3];
        }
        // ---- O += P V~: the score accumulators of two key n-tiles are the A fragment of one 16-key step
#pragma unroll
        for (int ks = 0; ks < AP_BN / 16; ++ks) {
            uint32_t pa[4];
            pa[0] = pack_h2(s[2 * ks][0], s[2 * ks][1]);
            pa[1] = pack_h2(s[2 * ks][2], s[2 * ks][3]);
            pa[2] = pack_h2(s[2 * ks + 1][0], s[2 * ks + 1][1]);
            pa[3] = pack_h2(s[2 * ks + 1][2], s[2 * ks + 1][3]);
#pragma unroll
            for (int d = 0; d < DT; ++d) {
                const half* bv = vt + (d * 8 + gq) * VP + ks * 16 + 2 * tig;
                mma16816(o[d], pa, *reinterpret_cast<const uint32_t*>(bv), *reinterpret_cast<const uint32_t*>(bv + 8));
            }
        }
        __syncthreads();                                  // kh / vt and the stage are free for the next tile
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");

    // ---- normalise, stage the rotated output tile in fp32, rotate back (x = H y / 32) and store
#pragma unroll
    for (int o2 = 1; o2 < 4; o2 <<= 1) {
        l0 += __shfl_xor_sync(0xffffffffu, l0, o2);
        l1 += __shfl_xor_sync(0xffffffffu, l1, o2);
    }
    const float i0 = (1.0f / 32.0f) / l0, i1 = (1.0f / 32.0f) / l1;
#pragma unroll
    for (int d = 0; d < DT; ++d) {
        *reinterpret_cast<float2*>(os + r0 * OP + d * 8 + 2 * tig) = make_float2(o[d][0] * i0, o[d][1] * i0);
        *reinterpret_cast<float2*>(os + (r0 + 8) * OP + d * 8 + 2 * tig) = make_float2(o[d][2] * i1, o[d][3] * i1);
    }
    __syncthreads();
    for (int job = warp; job < AP_BM * UNITS; job += AP_WARPS) {
        const int r = job / UNITS, un = job - r * UNITS, R = m0 + r;
        if (R >= rows) break;                             // (warp-uniform: rows only grow with job)
        const float2 w = hadamard32_f(*reinterpret_cast<const float2*>(os + r * OP + un * 64 + 2 * lane), lane);
        const int t = R / g, h = kvh * g + (R - t * g);
        reinterpret_cast<half2*>(P.out + (((size_t)b * P.q_len + t) * P.H + h) * HD + un * 64)[lane] = __floats2half2_rn(w.x, w.y);
    }
}

template <int HD, int KB, int VB>
static int prefill_launch(dim3 grid, size_t smem, cudaStream_t stream, const PrefillParams& P) {
    static bool attr_set[64] = {false};
    int dev = 0;
    EXL2B_CUDA(cudaGetDevice(&dev));
    if (!attr_set[dev]) {
        EXL2B_CUDA(cudaFuncSetAttribute(attn_prefill_kernel<HD, KB, VB>, cudaFuncAttributeMaxDynamicSharedMemorySize, AP_SMEM_MAX));
        attr_set[dev] = true;
    }
    EXL2B_CUDA(launch_pdl_f("attn", attn_prefill_kernel<HD, KB, VB>, grid, dim3(AP_THREADS), smem, stream, P));
    return 0;
}

template <int KB, int VB>
static int prefill_launch_hd(int head_dim, dim3 grid, size_t smem, cudaStream_t stream, const PrefillParams& P) {
    if (head_dim == 128) return prefill_launch<128, KB, VB>(grid, smem, stream, P);
    return prefill_launch<64, KB, VB>(grid, smem, stream, P);
}

}  // namespace exl2b

using namespace exl2b;

extern "C" int exl2b_paged_attn_prefill_q(const uint16_t* q, const uint16_t* k_new, const uint16_t* v_new, uint8_t* k_cache,
                                          uint16_t* k_scales, uint8_t* v_cache, uint16_t* v_scales, const int32_t* cache_seqlens,
                                          const int32_t* block_table, uint16_t* out, int batch, int q_len, int num_heads,
                                          int num_kv_heads, int head_dim, int page_size, int pages_per_seq, float softmax_scale,
                                          int wbits, exl2b_stream_t stream) {
    // every argument check comes before the first CUDA call
    EXL2B_REQUIRE(q && k_new && v_new && k_cache && k_scales && v_cache && v_scales && cache_seqlens && block_table && out, "null argument");
    EXL2B_REQUIRE(wbits == 4 || wbits == 6 || wbits == 8, "cache wbits must be 4 (Q4), 6 (Q6) or 8 (Q8); got %d", wbits);
    const int kb = wbits == 4 ? 4 : 8, vb = wbits == 8 ? 8 : 4;
    EXL2B_REQUIRE(head_dim == 64 || head_dim == 128, "head_dim %d not supported (64 or 128)", head_dim);
    EXL2B_REQUIRE(num_heads > 0 && num_kv_heads > 0 && num_heads % num_kv_heads == 0,
                  "bad GQA ratio: %d query heads over %d kv heads", num_heads, num_kv_heads);
    EXL2B_REQUIRE(page_size > 0 && page_size % AP_BN == 0, "page_size %d is not a multiple of the %d-position key tile", page_size, AP_BN);
    EXL2B_REQUIRE(pages_per_seq > 0 && (long)pages_per_seq * page_size <= INT32_MAX, "bad pages_per_seq %d", pages_per_seq);
    const PrefillSmem m = prefill_smem_map(head_dim, kb, vb, pages_per_seq);
    EXL2B_REQUIRE(m.total <= (uint32_t)AP_SMEM_MAX, "prompt attention needs %u bytes of shared memory for a page table of %d pages, "
                  "over the limit of %d", m.total, pages_per_seq, AP_SMEM_MAX);
    EXL2B_REQUIRE(batch >= 1 && batch <= 65535 && q_len >= 1 && num_kv_heads <= 65535, "bad shape: batch %d, q_len %d", batch, q_len);
    const long rows = (long)q_len * (num_heads / num_kv_heads);
    EXL2B_REQUIRE((rows + AP_BM - 1) / AP_BM <= INT32_MAX, "q_len %d too large", q_len);
    PrefillParams P = {};
    P.q = (const half*)q; P.k_new = (const half*)k_new; P.v_new = (const half*)v_new;
    P.k_q = k_cache; P.k_s = (half*)k_scales; P.v_q = v_cache; P.v_s = (half*)v_scales;
    P.cache_seqlens = cache_seqlens; P.block_table = block_table; P.out = (half*)out;
    P.q_len = q_len; P.H = num_heads; P.KVH = num_kv_heads; P.group = num_heads / num_kv_heads;
    P.page_size = page_size; P.pages_per_seq = pages_per_seq; P.max_ctx = page_size * pages_per_seq;
    P.scale_log2 = softmax_scale * 1.4426950408889634f;
    int dev = 0;
    EXL2B_CUDA(cudaGetDevice(&dev));
    EXL2B_REQUIRE(dev >= 0 && dev < 64, "bad device");
    int rc = attn_err_flag(dev, &P.err);
    if (rc) return rc;
    const dim3 grid((unsigned)((rows + AP_BM - 1) / AP_BM), (unsigned)num_kv_heads, (unsigned)batch);
    if (wbits == 4) return prefill_launch_hd<4, 4>(head_dim, grid, m.total, (cudaStream_t)stream, P);
    if (wbits == 6) return prefill_launch_hd<8, 4>(head_dim, grid, m.total, (cudaStream_t)stream, P);
    return prefill_launch_hd<8, 8>(head_dim, grid, m.total, (cudaStream_t)stream, P);
}
