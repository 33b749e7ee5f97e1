// LoRA adapters on the fused attention / MLP blocks: y_P += (in_P · A) · B for every active adapter of a projection P
// (reference: cuda/lora.cu, applied in q_attn.cu:266-300 and q_mlp.cu:183-236 as two cuBLAS HGEMMs per adapter).
//
// One launch per adapted STAGE -- q|k|v, o, gate|up, down -- serves every active adapter of every projection in it.  Projections
// of a stage share their input, so their A columns are stacked into one [K, R] operand (R = the stage's ranks, each rounded up to
// 8) and all of x·A is one product.  The launch is a grid of thread-block clusters (LORA_CLUSTER CTAs):
//   1. the cluster's CTAs split K; each stages its slice of the input rows in shared memory (with the RMSNorm weight applied and
//      the sums of squares taken, for q|k|v and gate|up, whose inputs are the block's normed rows) and computes a partial x·A
//      for all rows of its row tile and all R stacked columns;
//   2. every CTA sums the cluster's partials (and sums of squares) through distributed shared memory, in rank order, so all CTAs
//      of all clusters hold the same t = norm(x)·A;
//   3. each CTA applies its share of the stacked B columns, t·B, to the base GEMMs' outputs and finishes them: the residual stream
//      (o, down), RoPE of q and k (q|k|v), act(gate)·up (gate|up).
// The one-row form (LoraParams::one_row) serves the chained single-row decode step (blocks.cu, chained adapted calls): there the
// base launches write each output twice, as a plain row and as a copy in the next consumer's stored-row order, and every
// consumer forms RMSNorm, RoPE and act·mul itself.  So the LoRA launch only adds the deltas, to the plain row and to that copy
// (the mirror), and phase 3 spreads the columns over every CTA with 16-byte loads of B.  Down's input then is act(gate)·up
// formed from the two plain rows (LoraParams::x2).  A's rows and B's columns are requested into L2 before the dependency wait.
// Clusters split the output columns and recompute the small x·A from L2.  No global scratch, no atomics: the result is
// deterministic, and the adapter list travels by value in the kernel parameters, so the launch can be captured in a graph.
// All active adapters of a projection are summed in fp32 and y is rounded once (the reference rounds x·A to fp16 and y after
// each adapter).
#include <cooperative_groups.h>

#include <algorithm>

#include "lora.cuh"

namespace cg = cooperative_groups;

namespace exl2b {

constexpr int LORA_THREADS = 256;
constexpr int LORA_WARPS = LORA_THREADS / 32;
constexpr int LORA_CLUSTER = 8;                 // CTAs per cluster: the portable maximum
constexpr int LORA_MAX_CTAS = 128;              // at most one wave on the 132 SMs
constexpr int LORA_SMEM_MAX = 184 * 1024;       // staged input rows of a CTA's K slice (fp32), beside ~35 KB of static arrays

// adapter columns are stacked in groups of 8 (one 16-byte row segment of A per load): offsets and the bound count whole groups
__host__ __device__ inline int rank_slots(int rank) { return (rank + 7) & ~7; }

// outputs of a one-row launch: q, k, v / gate, up / the residual stream
__host__ __device__ inline int lora_outputs(int epi) { return epi == LORA_QKV ? 3 : epi == LORA_ADD_PAIR ? 2 : 1; }

// [p, p + bytes) into L2 at normal priority (the weights the GEMVs stream meanwhile are evict-first), shrunk to whole 16-byte
// units inside the range
__device__ __forceinline__ void prefetch_l2(const void* p, size_t bytes) {
    const uintptr_t a = ((uintptr_t)p + 15) & ~(uintptr_t)15, e = ((uintptr_t)p + bytes) & ~(uintptr_t)15;
    if (e > a) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(a), "r"((uint32_t)(e - a)) : "memory");
}

// one-row form: this CTA's groups [g0, g1) of 8 output columns, numbered over the launch's outputs in order
__device__ __forceinline__ void one_row_groups(const LoraParams& P, int& g0, int& g1) {
    const int gpc = (P.groups + (int)gridDim.x - 1) / (int)gridDim.x;
    g0 = min(P.groups, (int)blockIdx.x * gpc);
    g1 = min(P.groups, g0 + gpc);
}

// one-row form: the rows of B this CTA's columns read, one L2 prefetch per (segment, rank row) where B's rows are 16-byte aligned
__device__ void lora_prefetch_b(const LoraParams& P, int tid) {
    int g0, g1;
    one_row_groups(P, g0, g1);
    for (int p = 0, first = 0; p < lora_outputs(P.epi); ++p) {
        const int n = P.n[p], gp = (n + 7) >> 3;
        const int c0 = max(g0 - first, 0) * 8, c1 = min(min(g1 - first, gp) * 8, n);
        first += gp;
        if (c1 <= c0 || (n & 7)) continue;
        for (int s = 0; s < P.nseg; ++s) {
            const LoraSeg& sg = P.seg[s];
            if (sg.proj != p) continue;
            for (int j = tid; j < sg.rank; j += LORA_THREADS) prefetch_l2(sg.b + (size_t)j * n + c0, (size_t)(c1 - c0) * sizeof(half));
        }
    }
}

// ONE_ROW: LoraParams::one_row (a separate instantiation, so the un-chained form's code carries none of the one-row branches)
template <bool ONE_ROW>
__global__ void __launch_bounds__(LORA_THREADS) lora_kernel(const __grid_constant__ LoraParams P) {
    extern __shared__ float xs[];                          // [mt][len]: this CTA's K slice of the tile's input rows
    __shared__ float part[LORA_MT * LORA_MAX_RANK];        // this CTA's x·A over its slice, read by the whole cluster
    __shared__ float t_s[LORA_MT * LORA_MAX_RANK];         // the cluster's sum: norm(x)·A
    __shared__ float red[LORA_WARPS][LORA_MT * 8];         // warps that split one column group's K range
    __shared__ float ss_w[LORA_WARPS][LORA_MT];
    __shared__ float part_ss[LORA_MT];
    __shared__ float rs_s[LORA_MT];
    cg::cluster_group cluster = cg::this_cluster();
    const int cs = (int)cluster.num_blocks(), cr = (int)cluster.block_rank();
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int R = P.R, row0 = blockIdx.y * LORA_MT, mt = min(LORA_MT, P.rows - row0);
    const int kper = ((P.K + cs - 1) / cs + 7) & ~7;
    const int k0 = min(P.K, cr * kper), len = min(P.K, k0 + kper) - k0;

    // ---- 0. one-row form: the static operands, requested into L2 while the predecessor still runs: this CTA's rows of A and
    //      its columns of B ---------------------------------------------------------------------------------------------------------
    if constexpr (ONE_ROW) {
        if (tid < P.nseg) {
            const LoraSeg& sg = P.seg[tid];
            prefetch_l2(sg.a + (size_t)k0 * sg.rank, (size_t)len * sg.rank * sizeof(half));
        }
        lora_prefetch_b(P, tid);
    }
    griddep_launch_dependents();
    griddep_wait();

    // ---- 1. stage the input slice, sums of squares of the raw rows ------------------------------------------------------------
    float ss[LORA_MT];
#pragma unroll
    for (int m = 0; m < LORA_MT; ++m) {
        ss[m] = 0.f;
        if (m < mt) {
            const half* xr = P.x + (size_t)(row0 + m) * P.ldx + k0;
            const half* x2r = ONE_ROW && P.x2 ? P.x2 + (size_t)(row0 + m) * P.ldx + k0 : nullptr;
            for (int k = tid; k < len; k += LORA_THREADS) {
                float f;
                if (ONE_ROW && P.x2) f = __half2float(__hmul(P.gelu ? gelu1(xr[k]) : __low2half(silu2(__half2half2(xr[k]))), x2r[k]));
                else f = __half2float(xr[k]);
                ss[m] = fmaf(f, f, ss[m]);
                if (P.norm_w) f *= __half2float(P.norm_w[k0 + k]);
                xs[m * len + k] = f;
            }
        }
    }
#pragma unroll
    for (int m = 0; m < LORA_MT; ++m) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ss[m] += __shfl_xor_sync(0xffffffffu, ss[m], o);
        if (lane == 0) ss_w[warp][m] = ss[m];
    }
    __syncthreads();
    if (tid < LORA_MT) {
        float s = 0.f;
        for (int w = 0; w < LORA_WARPS; ++w) s += ss_w[w][tid];
        part_ss[tid] = s;
    }

    // ---- partial x·A: warps take column groups of 8; a group's K range is split over its lanes (and over several warps when
    //      there are fewer groups than warps) and reduced in a fixed order ---------------------------------------------------------
    const int groups = R >> 3;
    const int wpg = groups >= LORA_WARPS ? 1 : LORA_WARPS / groups;      // warps per group
    for (int grp = warp / wpg; grp < groups && warp < groups * wpg; grp += LORA_WARPS / wpg) {
        const int sub = warp % wpg, col = grp * 8;
        const LoraSeg* sg = nullptr;
        for (int s = 0; s < P.nseg; ++s)
            if (col >= P.seg[s].off && col < P.seg[s].off + rank_slots(P.seg[s].rank)) sg = &P.seg[s];
        float acc[LORA_MT][8];
#pragma unroll
        for (int m = 0; m < LORA_MT; ++m)
#pragma unroll
            for (int c = 0; c < 8; ++c) acc[m][c] = 0.f;
        if (sg) {
            const int c0 = col - sg->off, cnt = min(8, sg->rank - c0), rank = sg->rank;
            const half* a = sg->a + (size_t)k0 * rank + c0;
            const bool vec = cnt == 8 && (rank & 7) == 0 && ((uintptr_t)a & 15) == 0;
#pragma unroll 4
            for (int k = sub * 32 + lane; k < len; k += wpg * 32) {
                float av[8];
                if (vec) {
                    const uint4 w = ldg_ef(reinterpret_cast<const uint4*>(a + (size_t)k * rank));
                    const half2* h = reinterpret_cast<const half2*>(&w);
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        av[2 * i] = __low2float(h[i]);
                        av[2 * i + 1] = __high2float(h[i]);
                    }
                } else {
#pragma unroll
                    for (int c = 0; c < 8; ++c) av[c] = c < cnt ? __half2float(a[(size_t)k * rank + c]) : 0.f;
                }
#pragma unroll
                for (int m = 0; m < LORA_MT; ++m) {
                    if (m < mt) {
                        const float xv = xs[m * len + k];
#pragma unroll
                        for (int c = 0; c < 8; ++c) acc[m][c] = fmaf(xv, av[c], acc[m][c]);
                    }
                }
            }
        }
#pragma unroll
        for (int m = 0; m < LORA_MT; ++m)
#pragma unroll
            for (int c = 0; c < 8; ++c)
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) acc[m][c] += __shfl_xor_sync(0xffffffffu, acc[m][c], o);
#pragma unroll
        for (int e = 0; e < LORA_MT * 8; ++e) {
            if ((e & 31) == lane) {
                if (wpg == 1) part[(e >> 3) * R + col + (e & 7)] = acc[e >> 3][e & 7];
                else red[warp][e] = acc[e >> 3][e & 7];
            }
        }
    }
    __syncthreads();
    if (wpg > 1) {
        for (int i = tid; i < groups * LORA_MT * 8; i += LORA_THREADS) {
            const int grp = i / (LORA_MT * 8), e = i % (LORA_MT * 8);
            float s = 0.f;
            for (int w = 0; w < wpg; ++w) s += red[grp * wpg + w][e];
            part[(e >> 3) * R + grp * 8 + (e & 7)] = s;
        }
    }

    // ---- 2. the cluster's sum, in rank order ------------------------------------------------------------------------------------
    cluster.sync();
    if (tid < mt) {
        float s = 0.f;
        for (int r = 0; r < cs; ++r) s += cluster.map_shared_rank(part_ss, r)[tid];
        rs_s[tid] = P.norm_w ? rsqrtf(s * (1.0f / (float)P.K) + P.norm_eps) : 1.0f;
    }
    __syncthreads();
    for (int i = tid; i < mt * R; i += LORA_THREADS) {
        float s = 0.f;
        for (int r = 0; r < cs; ++r) s += cluster.map_shared_rank(part, r)[i];
        t_s[i] = s * rs_s[i / R];
    }
    cluster.sync();           // t_s complete; no CTA leaves while another still reads its partials

    // ---- 3, one-row form: groups of 8 columns, the rank rows of a group split between tpg adjacent lanes (16-byte loads of B),
    //      reduced by shuffles; the group's columns finished by its lanes in turn, each value stored to y and to its mirror -------
    if constexpr (ONE_ROW) {
        const int tpg = P.tpg;
        int g0, g1;
        one_row_groups(P, g0, g1);
        for (int base = 0; base < (g1 - g0) * tpg; base += LORA_THREADS) {      // the same trip count in every thread
            const int w = base + tid, g = g0 + w / tpg, sub = w & (tpg - 1);
            float d[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) d[e] = 0.f;
            int p = 0, c = 0;
            if (g < g1) {
                int gg = g;
                while (p < lora_outputs(P.epi) - 1 && gg >= (P.n[p] + 7) >> 3) gg -= (P.n[p++] + 7) >> 3;
                c = gg * 8;
                const int n = P.n[p];
                for (int s = 0, f0 = 0; s < P.nseg; ++s) {
                    const LoraSeg& sg = P.seg[s];
                    if (sg.proj != p) continue;
                    const half* b = sg.b + c;
                    const bool vec = (n & 7) == 0 && ((uintptr_t)sg.b & 15) == 0;
#pragma unroll 2
                    for (int j = (sub - f0) & (tpg - 1); j < sg.rank; j += tpg) {      // rank row f0 + j of the projection: lane sub
                        const float t = t_s[sg.off + j];
                        if (vec) {
                            const uint4 v = ldg_ef(reinterpret_cast<const uint4*>(b + (size_t)j * n));
                            const half2* h = reinterpret_cast<const half2*>(&v);
#pragma unroll
                            for (int i = 0; i < 4; ++i) {
                                d[2 * i] = fmaf(t, __low2float(h[i]), d[2 * i]);
                                d[2 * i + 1] = fmaf(t, __high2float(h[i]), d[2 * i + 1]);
                            }
                        } else {
#pragma unroll
                            for (int e = 0; e < 8; ++e)
                                if (c + e < n) d[e] = fmaf(t, __half2float(b[(size_t)j * n + e]), d[e]);
                        }
                    }
                    f0 += sg.rank;
                }
            }
            for (int o = tpg >> 1; o > 0; o >>= 1)
#pragma unroll
                for (int e = 0; e < 8; ++e) d[e] += __shfl_xor_sync(0xffffffffu, d[e], o);
            if (g >= g1) continue;
            half* y = P.y[p];
            half* mir = P.mirror[p];
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                if ((e & (tpg - 1)) != sub || c + e >= P.n[p]) continue;
                const half v = __float2half_rn(__half2float(y[c + e]) + d[e]);
                y[c + e] = v;
                if (mir) mir[P.mirror_invperm[p][c + e]] = v;
            }
        }
        return;
    }

    // ---- 3. t·B on this CTA's units of output columns, then the stage's epilogue -------------------------------------------------
    const int ctas = gridDim.x, upc = (P.units + ctas - 1) / ctas;
    const int u0 = blockIdx.x * upc, u1 = min(P.units, u0 + upc);
    for (int idx = u0 * P.unit_pairs + tid; idx < u1 * P.unit_pairs; idx += LORA_THREADS) {
        const int u = idx / P.unit_pairs, i = idx - u * P.unit_pairs;
        int pa, ca, pb, cb;
        bool rot = false;
        if (P.epi == LORA_QKV) {
            const int hd = P.head_dim;
            int h = u;
            pa = 0;
            if (h >= P.heads_q) { h -= P.heads_q; pa = 1; }
            if (pa == 1 && h >= P.heads_kv) { h -= P.heads_kv; pa = 2; }
            pb = pa;
            rot = P.sin && pa < 2;
            const int S = P.sincos_size, S2 = S >> 1;
            if (rot && P.neox) {
                if (i < S2) { ca = i; cb = i + S2; }
                else { ca = S + 2 * (i - S2); cb = ca + 1; rot = false; }
            } else {
                ca = 2 * i;
                cb = ca + 1;
                rot = rot && ca < S;
            }
            ca += h * hd;
            cb += h * hd;
        } else if (P.epi == LORA_ACT_MUL) {
            pa = 0; pb = 1;
            ca = cb = idx;
            if (ca >= P.n[0]) continue;
        } else {
            pa = pb = 0;
            ca = 2 * idx;
            cb = ca + 1;
            if (ca >= P.n[0]) continue;
        }
        float da[LORA_MT], db[LORA_MT];
#pragma unroll
        for (int m = 0; m < LORA_MT; ++m) da[m] = db[m] = 0.f;
        for (int s = 0; s < P.nseg; ++s) {
            const LoraSeg& sg = P.seg[s];
            if (sg.proj != pa && sg.proj != pb) continue;
            const int n = P.n[sg.proj];
            const half* b = sg.b;
#pragma unroll 4
            for (int j = 0; j < sg.rank; ++j) {
                const float* t = t_s + sg.off + j;
                const size_t rb = (size_t)j * n;
                if (sg.proj == pa) {
                    const float bv = __half2float(__ushort_as_half(ldg_ef(reinterpret_cast<const uint16_t*>(b + rb + ca))));
#pragma unroll
                    for (int m = 0; m < LORA_MT; ++m) if (m < mt) da[m] = fmaf(t[m * R], bv, da[m]);
                }
                if (sg.proj == pb) {
                    const float bv = __half2float(__ushort_as_half(ldg_ef(reinterpret_cast<const uint16_t*>(b + rb + cb))));
#pragma unroll
                    for (int m = 0; m < LORA_MT; ++m) if (m < mt) db[m] = fmaf(t[m * R], bv, db[m]);
                }
            }
        }
#pragma unroll
        for (int m = 0; m < LORA_MT; ++m) {
            if (m >= mt) continue;
            const int row = row0 + m;
            half* ya = P.y[pa] + (size_t)row * P.ldy[pa];
            half* yb = P.y[pb] + (size_t)row * P.ldy[pb];
            half va = __float2half_rn(__half2float(ya[ca]) + da[m]);
            half vb = __float2half_rn(__half2float(yb[cb]) + db[m]);
            if (P.epi == LORA_ACT_MUL) {
                const half act = P.gelu ? gelu1(va) : __low2half(silu2(__half2half2(va)));
                P.act_out[(size_t)row * P.ld_act + ca] = __hmul(act, vb);
                continue;
            }
            if (rot) {                       // rope_kernel, lane for lane (cuda/rope.cu:52-67,111-122)
                const int bb = row / P.q_len, tt = row - bb * P.q_len;
                int base = P.past_len;
                if (base == -1) base = max(P.past_lens[bb], 0);
                else if (P.past_lens) base += P.past_lens[bb];
                const size_t sr = (size_t)max(base + tt, 0) * P.sincos_size;
                const int d = ca % P.head_dim;
                if (P.neox) {
                    const half c = P.cos[sr + d], sn = P.sin[sr + d];
                    const half l = va, r = vb;
                    va = __hfma(l, c, __hmul(r, __hneg(sn)));
                    vb = __hfma(r, c, __hmul(l, sn));
                } else {
                    const half c0 = P.cos[sr + d], c1 = P.cos[sr + d + 1], s0 = P.sin[sr + d], s1 = P.sin[sr + d + 1];
                    const half x0 = va, x1 = vb;
                    va = __hfma(x1, __hneg(s0), __hmul(x0, c0));
                    vb = __hfma(x0, s1, __hmul(x1, c1));
                }
            }
            ya[ca] = va;
            yb[cb] = vb;
        }
    }
}

int lora_stack(const std::vector<LoraAdapter>& ads, const uint64_t* ids, int num_ids, const int* projs, int nproj, LoraParams& p) {
    p.nseg = 0;
    p.R = 0;
    for (int i = 0; i < num_ids; ++i) {
        const LoraAdapter* ad = nullptr;
        for (const LoraAdapter& a : ads)
            if (a.id == ids[i]) ad = &a;
        if (!ad) continue;                                   // registered nowhere on this handle (lora.cu:20-21)
        for (int j = 0; j < nproj; ++j) {
            const LoraProj& lp = ad->p[projs[j]];
            if (!lp.a) continue;
            EXL2B_REQUIRE(p.nseg < LORA_MAX_SEGS, "LoRA: more than %d (adapter, projection) pairs in one launch", LORA_MAX_SEGS);
            EXL2B_REQUIRE(p.R + rank_slots(lp.rank) <= LORA_MAX_RANK,
                          "LoRA: the active adapters' ranks (each rounded up to 8) sum to more than %d on one stage "
                          "(EXL2B_LORA_MAX_RANK)", LORA_MAX_RANK);
            p.seg[p.nseg++] = LoraSeg{lp.a, lp.b, lp.rank, p.R, j, i};
            p.R += rank_slots(lp.rank);
        }
    }
    return 0;
}

int lora_take(const exl2b_lora_t* loras, int num, const int* ks, const int* ns, int nprojs, const int (*stages)[4], int nstages,
              std::vector<LoraAdapter>& out, int* max_rank) {
    EXL2B_REQUIRE(num >= 0 && (num == 0 || loras), "null argument");
    EXL2B_REQUIRE(num <= LORA_MAX_ADAPTERS, "LoRA: %d adapters given, a block holds at most %d (EXL2B_LORA_MAX_ADAPTERS)", num,
                  LORA_MAX_ADAPTERS);
    std::vector<LoraAdapter> ads;
    int mr = 0;
    for (int i = 0; i < num; ++i) {
        const exl2b_lora_t& l = loras[i];
        for (int j = 0; j < i; ++j) EXL2B_REQUIRE(loras[j].id != l.id, "LoRA: adapter id %llu given twice", (unsigned long long)l.id);
        LoraAdapter ad = {};
        ad.id = l.id;
        for (int p = 0; p < nprojs; ++p) {
            if (!l.a[p] && !l.b[p]) continue;
            EXL2B_REQUIRE(l.a[p] && l.b[p], "LoRA: adapter %llu has %s without %s on projection %d", (unsigned long long)l.id,
                          l.a[p] ? "A" : "B", l.a[p] ? "B" : "A", p);
            EXL2B_REQUIRE(l.rank[p] > 0 && rank_slots(l.rank[p]) <= LORA_MAX_RANK, "LoRA: rank %d is outside 1..%d (EXL2B_LORA_MAX_RANK)",
                          l.rank[p], LORA_MAX_RANK);
            EXL2B_REQUIRE(l.a_rows[p] == ks[p] && l.b_cols[p] == ns[p],
                          "LoRA: adapter %llu on projection %d is [%d, %d] x [%d, %d], the matrix is [%d, %d]", (unsigned long long)l.id,
                          p, l.a_rows[p], l.rank[p], l.rank[p], l.b_cols[p], ks[p], ns[p]);
            ad.p[p] = LoraProj{(const half*)l.a[p], (const half*)l.b[p], l.rank[p]};
            mr = std::max(mr, l.rank[p]);
        }
        ads.push_back(ad);
    }
    // every registered adapter may be active at once: the whole set must fit each stage's launch
    std::vector<uint64_t> ids;
    for (const LoraAdapter& a : ads) ids.push_back(a.id);
    for (int s = 0; s < nstages; ++s) {
        int np = 0;
        while (np < 4 && stages[s][np] >= 0) ++np;
        LoraParams p;
        int rc = lora_stack(ads, ids.data(), (int)ids.size(), stages[s], np, p);
        if (rc) return rc;
    }
    out.swap(ads);
    if (max_rank) *max_rank = mr;
    return 0;
}

int lora_launch(int device, cudaStream_t stream, LoraParams& p) {
    if (p.nseg == 0 || p.rows <= 0) return 0;
    int clusters = 0;
    if (p.one_row) {
        EXL2B_REQUIRE(p.rows == 1 && !p.sin && p.epi != LORA_ACT_MUL, "LoRA: the one-row form takes one row, no RoPE and no act·mul");
        // groups of 8 columns over up to one wave of CTAs; lanes per group while a CTA's groups fill its threads, at most the
        // largest summed rank of one projection
        p.groups = 0;
        int rmax = 0;
        for (int o = 0; o < lora_outputs(p.epi); ++o) {
            p.groups += (p.n[o] + 7) / 8;
            int r = 0;
            for (int s = 0; s < p.nseg; ++s) r += p.seg[s].proj == o ? p.seg[s].rank : 0;
            rmax = std::max(rmax, r);
        }
        clusters = std::max(1, std::min(LORA_MAX_CTAS / LORA_CLUSTER, (p.groups + LORA_CLUSTER - 1) / LORA_CLUSTER));
        const int gpc = (p.groups + clusters * LORA_CLUSTER - 1) / (clusters * LORA_CLUSTER);
        p.tpg = 1;
        while (p.tpg < 32 && p.tpg < rmax && 2 * p.tpg * gpc <= LORA_THREADS) p.tpg *= 2;
    } else if (p.epi == LORA_QKV) {
        p.unit_pairs = p.head_dim / 2;
        p.units = p.heads_q + 2 * p.heads_kv;
    } else if (p.epi == LORA_ACT_MUL) {
        p.unit_pairs = 64;
        p.units = (p.n[0] + 63) / 64;
    } else {
        EXL2B_REQUIRE(p.epi == LORA_ADD, "LoRA: epilogue %d needs the one-row form", p.epi);
        EXL2B_REQUIRE(p.n[0] % 2 == 0, "LoRA: output width %d is odd", p.n[0]);
        p.unit_pairs = 32;
        p.units = (p.n[0] + 63) / 64;
    }
    const int tiles = (p.rows + LORA_MT - 1) / LORA_MT;
    const int mt = std::min(LORA_MT, p.rows);
    const int kper = ((p.K + LORA_CLUSTER - 1) / LORA_CLUSTER + 7) & ~7;
    const size_t smem = (size_t)mt * kper * sizeof(float);
    EXL2B_REQUIRE(smem <= LORA_SMEM_MAX, "LoRA: input width %d needs %zu bytes of shared memory per CTA (at most %d)", p.K, smem,
                  LORA_SMEM_MAX);
    static bool attr_set[64] = {};
    if (!attr_set[device]) {
        EXL2B_CUDA(cudaFuncSetAttribute(lora_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, LORA_SMEM_MAX));
        EXL2B_CUDA(cudaFuncSetAttribute(lora_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, LORA_SMEM_MAX));
        attr_set[device] = true;
    }
    // clusters over the output units: up to one wave of CTAs in all, fewer when there are many row tiles
    const int want = (p.units + LORA_CLUSTER - 1) / LORA_CLUSTER;
    if (!p.one_row) clusters = std::max(1, std::min(want, LORA_MAX_CTAS / LORA_CLUSTER / tiles));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(clusters * LORA_CLUSTER, tiles);
    cfg.blockDim = dim3(LORA_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = LORA_CLUSTER;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_disabled("lora") ? 1 : 2;
    g_launch_count.fetch_add(1, std::memory_order_relaxed);
    EXL2B_CUDA(p.one_row ? cudaLaunchKernelEx(&cfg, lora_kernel<true>, p) : cudaLaunchKernelEx(&cfg, lora_kernel<false>, p));
    return 0;
}

}  // namespace exl2b

using namespace exl2b;

extern "C" int exl2b_lora_stack(const int* ranks, int num_adapters, int num_projs, int* seg_adapter, int* seg_proj, int* seg_off,
                                int* num_segs, int* total) {
    EXL2B_REQUIRE(ranks && seg_adapter && seg_proj && seg_off && num_segs && total, "null argument");
    EXL2B_REQUIRE(num_adapters >= 0 && num_adapters <= LORA_MAX_ADAPTERS && num_projs > 0 && num_projs <= 4, "bad argument");
    static const half dummy[8] = {};
    std::vector<LoraAdapter> ads(num_adapters);
    std::vector<uint64_t> ids(num_adapters);
    int projs[4];
    for (int j = 0; j < num_projs; ++j) projs[j] = j;
    for (int i = 0; i < num_adapters; ++i) {
        ads[i] = LoraAdapter{};
        ads[i].id = ids[i] = (uint64_t)i + 1;
        for (int j = 0; j < num_projs; ++j)
            if (ranks[i * num_projs + j] > 0) ads[i].p[j] = LoraProj{dummy, dummy, ranks[i * num_projs + j]};
    }
    LoraParams p;
    int rc = lora_stack(ads, ids.data(), num_adapters, projs, num_projs, p);
    if (rc) return rc;
    for (int s = 0; s < p.nseg; ++s) {
        seg_adapter[s] = p.seg[s].src;
        seg_proj[s] = p.seg[s].proj;
        seg_off[s] = p.seg[s].off;
    }
    *num_segs = p.nseg;
    *total = p.R;
    return 0;
}
