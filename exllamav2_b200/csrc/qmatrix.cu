// QMatrix creation: group bookkeeping, load-time re-pack into the private streaming layout (layout.h), and
// bit-exact reconstruct.  Replaces exllamav2_ext/cuda/q_matrix.cu (QMatrix::QMatrix :49-196, shuffle_kernel
// :21-44, make_sequential :555-680, reconstruct kernels :204-553).
#include <stdarg.h>
#include <string.h>

#include <algorithm>
#include <mutex>

#include "dequant.cuh"
#include "qmatrix.cuh"

namespace exl2b {

static thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launch_count{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int device_sm_count(int device) {
    static int cache[64] = {0};
    if (device < 0 || device >= 64) return 148;
    if (!cache[device]) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || n <= 0) n = 148;
        cache[device] = n;
    }
    return cache[device];
}

// ---- re-pack kernels -------------------------------------------------------------------------------------------
// One warp per (slab, strip, block).  Lane l gathers its 32 values from the checkpoint layout and writes its
// plane words.  Load-time only, so the gather is not tuned.

struct GroupInfo {   // per EXL2 group (device array)
    int bits;
    int first_qrow;   // first packed row in q_weight
    int row0;         // first stored k row
};

// byte offset of block `blk` of slab (tab.x) of `strip` for either layout
__device__ __forceinline__ size_t block_offset(int layout, int strip, int blk, uint32_t tab_x, int bits, uint32_t strip_bytes,
                                               uint32_t blk_stream_bytes) {
    return layout == LAYOUT_TC ? (size_t)strip * strip_bytes + (size_t)blk * blk_stream_bytes + tab_x
                               : (size_t)strip * strip_bytes + tab_x + (size_t)blk * block_bytes(bits);
}

__global__ void repack_exl2_kernel(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst, int N, int KS,
                                   const uint2* __restrict__ slab_tab, const GroupInfo* __restrict__ ginfo,
                                   uint32_t strip_bytes, uint32_t blk_stream_bytes, int layout) {
    const int ks = blockIdx.x, strip = blockIdx.y;
    const int blk = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint2 tab = slab_tab[ks];
    const GroupInfo gi = ginfo[tab.y & 0xFFFFu];
    const int bits = gi.bits;
    uint32_t vals[32];
#pragma unroll 4
    for (int i = 0; i < 32; ++i) {
        const ValuePos vp = value_pos_l(layout, lane, i);
        const int n = strip * strip_n(layout) + blk * BLOCK_N + vp.n_local;
        const int r = ks * SLAB_K + vp.k_local - gi.row0;
        const int bitpos = r * bits;
        const int word = gi.first_qrow + (bitpos >> 5), sh = bitpos & 31;
        uint32_t v = 0;
        if (n < N) {
            v = src[(size_t)word * N + n] >> sh;
            if (sh + bits > 32) v |= src[(size_t)(word + 1) * N + n] << (32 - sh);
            v &= (1u << bits) - 1u;
        }
        vals[i] = v;
    }
    uint32_t mw[8], ew[4];
    compose_lane_words(bits, vals, mw, ew);
    uint32_t* bp = dst + block_offset(layout, strip, blk, tab.x, bits, strip_bytes, blk_stream_bytes) / 4;
    const int Pm = plane_main(bits), Pe = plane_extra(bits);
    for (int w = 0; w < Pm; ++w) bp[main_word_index(bits, lane, w)] = mw[w];
    for (int w = 0; w < Pe; ++w) bp[extra_word_index(bits, lane, w)] = ew[w];
}

__global__ void repack_gptq_kernel(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst, int N, int KS,
                                   const uint16_t* __restrict__ perm, uint32_t strip_bytes, uint32_t blk_stream_bytes, int layout) {
    const int ks = blockIdx.x, strip = blockIdx.y;
    const int blk = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t vals[32];
#pragma unroll 4
    for (int i = 0; i < 32; ++i) {
        const ValuePos vp = value_pos_l(layout, lane, i);
        const int n = strip * strip_n(layout) + blk * BLOCK_N + vp.n_local;
        const int kp = ks * SLAB_K + vp.k_local;
        const int row = perm ? (int)perm[kp] : kp;    // stored row k' <- checkpoint row perm[k'] (make_sequential)
        uint32_t v = 0;
        if (n < N) v = (src[(size_t)(row >> 3) * N + n] >> ((row & 7) * 4)) & 15u;
        vals[i] = v;
    }
    uint32_t mw[8], ew[4];
    compose_lane_words(4, vals, mw, ew);
    const uint32_t tab_x = (uint32_t)ks * (layout == LAYOUT_TC ? block_bytes(4) : slab_bytes(4));
    uint32_t* bp = dst + block_offset(layout, strip, blk, tab_x, 4, strip_bytes, blk_stream_bytes) / 4;
    for (int w = 0; w < 4; ++w) bp[main_word_index(4, lane, w)] = mw[w];
}

// ---- reconstruct -------------------------------------------------------------------------------------------------
// One warp per (slab, strip, block): unpack in the fp16 domain (exact integers), one fp16 multiply by the fp16
// scale, scatter to out[perm[k'], n]  -- the same two roundings-free steps + one rounding as the reference
// (cuda/q_matrix.cu:389-412 EXL2; :283-303 GPTQ), hence bit-exact.

template <int BITS>
__device__ __forceinline__ void load_block_words(const uint32_t* bp, int lane, uint32_t* mw, uint32_t* ew) {
    constexpr int Pm = plane_main(BITS), Pe = plane_extra(BITS);
#pragma unroll
    for (int w = 0; w < Pm; ++w) mw[w] = bp[main_word_index(BITS, lane, w)];
#pragma unroll
    for (int w = 0; w < Pe; ++w) ew[w] = bp[extra_word_index(BITS, lane, w)];
}

__device__ __forceinline__ half exl2_scale_h(uint32_t nib, half smax) {
    const int q = (int)nib + 1;
    return __hmul(__int2half_rn(q * q), smax);     // dq_scale, cuda/quant/qdq_util.cuh:24-30
}

template <int BITS>
__device__ void reconstruct_block_exl2(const QMatView& v, const uint32_t* bp, int lane, int group, int n0, int k0,
                                       half* __restrict__ out, int ld, int col0) {
    uint32_t mw[8], ew[4], A[16];
    load_block_words<BITS>(bp, lane, mw, ew);
    dequant_block_exl2<BITS>(mw, ew, A);
    const half smax = v.q_scale_max[group];
#pragma unroll
    for (int p = 0; p < 16; ++p) {
        const int n = n0 + value_pos_l(v.layout, lane, p * 2).n_local;
        if (n >= v.N) continue;
        const uint32_t word = v.q_scale[(size_t)group * (v.N / 8) + (n >> 3)];
        const half s = exl2_scale_h((word >> ((n & 7) * 4)) & 15u, smax);
        const half2 w2 = __hmul2(*reinterpret_cast<const half2*>(&A[p]), __half2half2(s));
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int kp = k0 + value_pos_l(v.layout, lane, p * 2 + e).k_local;
            const int row = v.perm ? (int)v.perm[kp] : kp;
            out[(size_t)row * ld + (n - col0)] = e ? __high2half(w2) : __low2half(w2);
        }
    }
}

// Dense scale table of the batch-1 GEMV: one entry per (group, column), natural column order, so that its per-group flush is
// one coalesced load per warp with no nibble extraction / region lookup (EXL2: the exact fp16 dq_scale of
// cuda/quant/qdq_util.cuh:24-30; GPTQ: the checkpoint's fp16 scale and qzero + 1 of q_gemm_kernel_gptq.cuh:167-172).
__global__ void scale_table_kernel(QMatView v, void* __restrict__ out) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)v.groups * v.N) return;
    const int g = (int)(idx / v.N), n = (int)(idx - (size_t)g * v.N);
    if (!v.is_gptq) {
        const uint32_t word = v.q_scale[(size_t)g * (v.N / 8) + (n >> 3)];
        reinterpret_cast<half*>(out)[idx] = exl2_scale_h((word >> ((n & 7) * 4)) & 15u, v.q_scale_max[g]);
    } else {
        const uint32_t word = v.qzeros[(size_t)g * (v.N / 8) + (n >> 3)];
        const uint32_t zero = ((word >> ((n & 7) * 4)) & 15u) + 1u;
        reinterpret_cast<uint32_t*>(out)[idx] = (uint32_t)__half_as_ushort(v.gptq_scales[idx]) | (zero << 16);
    }
}

// out[row * ld + (n - col0)] for the strips [strip0, strip0 + gridDim.y): the whole matrix (ld = N, col0 = 0, strip0 = 0) for
// exl2b_reconstruct, or a column window for the large-M path (gemm_big.cu)
__global__ void reconstruct_kernel(QMatView v, int gptq_groupsize, half* __restrict__ out, int ld, int col0, int strip0) {
    const int ks = blockIdx.x, strip = strip0 + blockIdx.y;
    const int blk = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint2 tab = v.slab_tab[ks];
    const int bits = (tab.y >> 16) & 0xF, group = tab.y & 0xFFFF;
    const uint32_t* bp = v.packed + block_offset(v.layout, strip, blk, tab.x, bits, v.strip_bytes, v.blk_stream_bytes) / 4;
    const int n0 = strip * strip_n(v.layout) + blk * BLOCK_N, k0 = ks * SLAB_K;
    if (!v.is_gptq) {
        switch (bits) {
            case 2: reconstruct_block_exl2<2>(v, bp, lane, group, n0, k0, out, ld, col0); break;
            case 3: reconstruct_block_exl2<3>(v, bp, lane, group, n0, k0, out, ld, col0); break;
            case 4: reconstruct_block_exl2<4>(v, bp, lane, group, n0, k0, out, ld, col0); break;
            case 5: reconstruct_block_exl2<5>(v, bp, lane, group, n0, k0, out, ld, col0); break;
            case 6: reconstruct_block_exl2<6>(v, bp, lane, group, n0, k0, out, ld, col0); break;
            case 8: reconstruct_block_exl2<8>(v, bp, lane, group, n0, k0, out, ld, col0); break;
        }
    } else {
        uint32_t mw[8], ew[4];
        load_block_words<4>(bp, lane, mw, ew);
#pragma unroll
        for (int p = 0; p < 16; ++p) {
            const int n = n0 + value_pos_l(v.layout, lane, p * 2).n_local;
            if (n >= v.N) continue;
            const int z1 = (int)((v.qzeros[(size_t)group * (v.N / 8) + (n >> 3)] >> ((n & 7) * 4)) & 15u) + 1;
            const half sc = v.gptq_scales[(size_t)group * v.N + n];
            const int jm = pair_slot(4, p);
            const uint32_t x = mw[pair_word(4, p)] >> field_sh(4, jm);
            const uint32_t tm = and_or(x, field_mask(4, jm), field_magic(4, jm));
            const half2 c2 = __half2half2(__int2half_rn(-((1 << field_exp(4, jm)) + z1)));
            const uint32_t qz = h2add_bits(tm, *reinterpret_cast<const uint32_t*>(&c2));       // q - (zero + 1), exact
            const half2 w2 = __hmul2(__half2half2(sc), *reinterpret_cast<const half2*>(&qz));
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int kp = k0 + value_pos_l(v.layout, lane, p * 2 + e).k_local;
                const int row = v.perm ? (int)v.perm[kp] : kp;
                out[(size_t)row * ld + (n - col0)] = e ? __high2half(w2) : __low2half(w2);
            }
        }
    }
}

// ---- host side ---------------------------------------------------------------------------------------------------

static int build_tables_exl2(const exl2b_qmatrix_desc* d, const uint16_t* hg, std::vector<uint2>& tab,
                             std::vector<GroupInfo>& ginfo, uint32_t& bits_mask, uint32_t& strip_bytes, int layout) {
    const int G = d->groups, K = d->height;
    ginfo.resize(G);
    int row = 0;
    for (int i = 0; i < G; ++i) {
        const int bits = hg[2 * i];
        EXL2B_REQUIRE(bits_supported(bits), "EXL2 group %d has unsupported bit width %d", i, bits);
        int rows;
        if (i < G - 1) {
            const int qrows = (int)hg[2 * i + 3] - (int)hg[2 * i + 1];
            rows = qrows * 32 / bits;          // q_matrix.cu:141-145
        } else {
            rows = K - row;                    // q_matrix.cu:148
        }
        EXL2B_REQUIRE(rows > 0 && rows % SLAB_K == 0, "EXL2 group %d covers %d rows; multiples of 32 are required", i, rows);
        ginfo[i] = GroupInfo{bits, (int)hg[2 * i + 1], row};
        bits_mask |= 1u << bits;
        row += rows;
    }
    EXL2B_REQUIRE(row == K, "EXL2 groups cover %d rows but height is %d", row, K);
    const int KS = K / SLAB_K;
    tab.resize(KS);
    uint32_t off = 0;
    int gi = 0;
    for (int ks = 0; ks < KS; ++ks) {
        while (gi + 1 < G && ks * SLAB_K >= ginfo[gi + 1].row0) gi++;
        tab[ks].x = off;
        tab[ks].y = (uint32_t)gi | ((uint32_t)ginfo[gi].bits << 16);
        off += (layout == LAYOUT_TC) ? block_bytes(ginfo[gi].bits) : slab_bytes(ginfo[gi].bits);
    }
    strip_bytes = off;      // MMA: bytes of a strip;  TC: bytes of one block stream (caller multiplies by 4)
    return 0;
}

// Group structure -> at most MAX_REGIONS arithmetic regions (same bits, same power-of-two group size; a short last
// group may close a region).  Converter output always fits (conversion/qparams.py: <= 3 bit widths per matrix).
static int build_regions(QMatView& v, const std::vector<uint2>& tab, const std::vector<int>& group_rows) {
    v.num_regions = 0;
    int ks = 0;
    const int KS = v.KS;
    while (ks < KS) {
        const int bits = (tab[ks].y >> 16) & 0xF, g0 = tab[ks].y & 0xFFFF;
        const int rows = group_rows[g0];
        int spg = rows / SLAB_K, lg = 0;
        while ((1 << lg) < spg) ++lg;
        EXL2B_REQUIRE((1 << lg) == spg || g0 == v.groups - 1, "group of %d rows: group sizes must be 32 * 2^n", rows);
        EXL2B_REQUIRE(v.num_regions < MAX_REGIONS, "more than %d (bits, group size) regions in one matrix", MAX_REGIONS);
        QRegion& r = v.reg[v.num_regions++];
        r.ks_begin = ks;
        r.bits = bits;
        r.spg_log2 = lg;
        r.group_base = g0;
        r.off_base = tab[ks].x;
        // extend while groups keep the same bits and size (the last group of the matrix may be shorter)
        int g = g0;
        while (ks < KS) {
            const int gg = tab[ks].y & 0xFFFF;
            if (gg != g) {
                const int b2 = (tab[ks].y >> 16) & 0xF, rows2 = group_rows[gg];
                const bool same = b2 == bits && (rows2 == rows || (gg == v.groups - 1 && rows2 < rows));
                if (!same || gg != g + 1) break;
                g = gg;
            }
            ++ks;
        }
    }
    return 0;
}

static void fill_left_same(std::vector<uint2>& tab) {
    const int KS = (int)tab.size();
    int left = 0;
    for (int ks = KS - 1; ks >= 0; --ks) {   // slabs left (incl. this one) with the same bit width
        const uint32_t b = (tab[ks].y >> 16) & 0xF;
        left = (ks + 1 < KS && ((tab[ks + 1].y >> 16) & 0xF) == b) ? left + 1 : 1;
        tab[ks].y |= (uint32_t)std::min(left, 4095) << 20;
    }
}

}  // namespace exl2b

using namespace exl2b;

extern "C" const char* exl2b_last_error(void) { return g_err; }
extern "C" int exl2b_version(void) { return 101; }
extern "C" uint64_t exl2b_launch_count(void) { return g_launch_count.load(); }

extern "C" int exl2b_make_group_map(const int16_t* q_groups, int num_groups, int num_qrows, int16_t* out,
                                    int out_capacity, int* k) {
    int n = 0;
    for (int i = 0; i < num_groups; ++i) {
        const int bits = q_groups[2 * i];
        EXL2B_REQUIRE(bits > 0, "bad q_groups");
        const int qrows = (i < num_groups - 1 ? q_groups[2 * i + 3] : num_qrows) - q_groups[2 * i + 1];
        const int rows = qrows * 32 / bits;
        for (int j = 0; j < rows; ++j) {
            EXL2B_REQUIRE(2 * n + 1 < out_capacity, "group map capacity %d too small", out_capacity);
            out[2 * n] = (int16_t)i;
            out[2 * n + 1] = (int16_t)(rows - j);
            ++n;
        }
    }
    if (k) *k = n;
    return 0;
}

extern "C" int exl2b_qmatrix_create(const exl2b_qmatrix_desc* d, exl2b_stream_t stream_, exl2b_qmatrix_t* out) {
    cudaStream_t stream = (cudaStream_t)stream_;
    EXL2B_REQUIRE(d && out, "null argument");
    EXL2B_REQUIRE(d->q_weight, "q_weight is NULL");
    const bool is_gptq = d->gptq_qzeros != nullptr;
    EXL2B_REQUIRE(is_gptq || (d->q_scale && d->q_scale_max && d->q_groups), "neither EXL2 nor GPTQ tensors given");
    EXL2B_REQUIRE(d->height > 0 && d->height % SLAB_K == 0, "height %d must be a positive multiple of 32", d->height);
    EXL2B_REQUIRE(d->width > 0 && d->width % 8 == 0, "width %d must be a positive multiple of 8", d->width);
    EXL2B_REQUIRE(d->height <= 65536, "height %d exceeds the 16-bit permutation range", d->height);
    EXL2B_CUDA(cudaSetDevice(d->device));

    QMatrix* m = new QMatrix();
    m->device = d->device;
    QMatView& v = m->v;
    v.layout = LAYOUT_TC;       // one layout serves every kernel (layout.h); the round-1 mma.sync layout is kept only as layout algebra
    v.K = d->height;
    v.N = d->width;
    v.KS = v.K / SLAB_K;
    v.strips = (v.N + strip_n(v.layout) - 1) / strip_n(v.layout);
    v.groups = d->groups;
    v.is_gptq = is_gptq ? 1 : 0;
    v.q_scale = d->q_scale;
    v.q_scale_max = (const half*)d->q_scale_max;
    v.qzeros = d->gptq_qzeros;
    v.gptq_scales = (const half*)d->gptq_scales;
    v.perm = d->q_perm;
    v.bias = (const half*)d->bias;
    m->invperm = d->q_perm ? d->q_invperm : nullptr;

    std::vector<GroupInfo> ginfo;
    int gptq_gs = 0;
    auto fail = [&](int code) { delete m; return code; };

    if (!is_gptq) {
        std::vector<uint16_t> hg(2 * (size_t)d->groups);
        if (cudaMemcpy(hg.data(), d->q_groups, hg.size() * 2, cudaMemcpyDefault) != cudaSuccess) {
            set_error("copying q_groups failed: %s", cudaGetErrorString(cudaGetLastError()));
            return fail(-1);
        }
        int rc = build_tables_exl2(d, hg.data(), m->slab_tab_host, ginfo, m->bits_mask, v.strip_bytes, v.layout);
        if (rc) return fail(rc);
        v.blk_stream_bytes = v.strip_bytes;
        if (v.layout == LAYOUT_TC) v.strip_bytes *= 4;
        std::vector<int> group_rows(d->groups);
        for (int i = 0; i < d->groups; ++i) group_rows[i] = (i + 1 < d->groups ? ginfo[i + 1].row0 : v.K) - ginfo[i].row0;
        rc = build_regions(v, m->slab_tab_host, group_rows);
        if (rc) return fail(rc);
        fill_left_same(m->slab_tab_host);
        const uint64_t expect_rows = (uint64_t)v.strip_bytes / (v.layout == LAYOUT_TC ? 512 : 256);   // sum over slabs of bits == packed rows
        if (d->q_weight_rows && (uint64_t)d->q_weight_rows != expect_rows) {
            set_error("q_weight has %d rows, groups imply %llu", d->q_weight_rows, (unsigned long long)expect_rows);
            return fail(-2);
        }
    } else {
        gptq_gs = 1;
        while (gptq_gs * d->groups < d->height) gptq_gs *= 2;      // q_matrix.cu:101-105
        if (gptq_gs % SLAB_K) { set_error("GPTQ group size %d must be a multiple of 32", gptq_gs); return fail(-2); }
        m->bits_mask = 1u << 4;
        m->slab_tab_host.resize(v.KS);
        for (int ks = 0; ks < v.KS; ++ks) {
            m->slab_tab_host[ks].x = (uint32_t)ks * (v.layout == LAYOUT_TC ? block_bytes(4) : slab_bytes(4));
            m->slab_tab_host[ks].y = (uint32_t)(ks * SLAB_K / gptq_gs) | (4u << 16) | ((uint32_t)std::min(v.KS - ks, 4095) << 20);
        }
        v.blk_stream_bytes = (uint32_t)v.KS * block_bytes(4);
        v.strip_bytes = (uint32_t)v.KS * block_bytes(4) * strip_blocks(v.layout);
        {
            int lg = 0;
            while ((SLAB_K << lg) < gptq_gs) ++lg;
            if ((SLAB_K << lg) != gptq_gs) { set_error("GPTQ group size %d must be 32 * 2^n", gptq_gs); return fail(-2); }
            v.num_regions = 1;
            v.reg[0] = QRegion{0, 4, lg, 0, 0u};
        }
        // act-order: stable group-sorted permutation, q_matrix.cu:597-647
        if (d->gptq_g_idx) {
            if (!d->q_perm || !d->q_invperm) { set_error("act-order GPTQ needs q_perm/q_invperm buffers"); return fail(-2); }
            const int K = v.K, G = d->groups;
            std::vector<uint32_t> start(G + 1, 0);
            for (int i = 0; i < K; ++i) {
                if (d->gptq_g_idx[i] < 0 || d->gptq_g_idx[i] >= G) { set_error("g_idx[%d] out of range", i); return fail(-2); }
                start[d->gptq_g_idx[i] + 1]++;
            }
            for (int i = 0; i < G; ++i) start[i + 1] += start[i];
            std::vector<uint16_t> perm(K), inv(K);
            for (int row = 0; row < K; ++row) {
                const uint32_t target = start[d->gptq_g_idx[row]]++;
                inv[row] = (uint16_t)target;
                perm[target] = (uint16_t)row;
            }
            if (cudaMemcpyAsync(d->q_perm, perm.data(), K * 2, cudaMemcpyHostToDevice, stream) != cudaSuccess ||
                cudaMemcpyAsync(d->q_invperm, inv.data(), K * 2, cudaMemcpyHostToDevice, stream) != cudaSuccess ||
                cudaStreamSynchronize(stream) != cudaSuccess) {
                set_error("uploading GPTQ permutation failed");
                return fail(-1);
            }
        }
    }

    // device tables
    const size_t tab_bytes = m->slab_tab_host.size() * sizeof(uint2);
    const size_t gi_bytes = ginfo.size() * sizeof(GroupInfo);
    if (cudaMalloc(&m->tables, tab_bytes + gi_bytes + 16) != cudaSuccess) { set_error("CUDA out of memory (tables)"); return fail(-3); }
    cudaMemcpyAsync(m->tables, m->slab_tab_host.data(), tab_bytes, cudaMemcpyHostToDevice, stream);
    GroupInfo* d_ginfo = (GroupInfo*)((char*)m->tables + tab_bytes);
    if (gi_bytes) cudaMemcpyAsync(d_ginfo, ginfo.data(), gi_bytes, cudaMemcpyHostToDevice, stream);
    v.slab_tab = (const uint2*)m->tables;

    // re-pack: write the private layout into a temp buffer, then back over q_weight (in place, like the
    // reference's shuffle) when the sizes match; keep the padded copy otherwise.
    m->packed_bytes = (uint64_t)v.strips * v.strip_bytes;
    uint32_t* tmp = nullptr;
    if (cudaMalloc(&tmp, m->packed_bytes) != cudaSuccess) {
        cudaFree(m->tables);
        set_error("CUDA out of memory");        // same message as the reference (ext_qmatrix.cpp:108)
        return fail(-3);
    }
    dim3 grid(v.KS, v.strips), block(32 * strip_blocks(v.layout));
    if (!is_gptq)
        repack_exl2_kernel<<<grid, block, 0, stream>>>(d->q_weight, tmp, v.N, v.KS, v.slab_tab, d_ginfo, v.strip_bytes,
                                                       v.blk_stream_bytes, v.layout);
    else
        repack_gptq_kernel<<<grid, block, 0, stream>>>(d->q_weight, tmp, v.N, v.KS, v.perm, v.strip_bytes, v.blk_stream_bytes,
                                                       v.layout);
    g_launch_count++;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) {
        if (v.N % strip_n(v.layout) == 0) {
            e = cudaMemcpyAsync(d->q_weight, tmp, m->packed_bytes, cudaMemcpyDeviceToDevice, stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
            cudaFree(tmp);
            v.packed = d->q_weight;
        } else {
            e = cudaStreamSynchronize(stream);
            m->owned_packed = tmp;
            v.packed = tmp;
        }
    }
    if (e != cudaSuccess) {
        set_error("re-pack failed: %s", cudaGetErrorString(e));
        cudaFree(m->tables);
        return fail(-1);
    }
    {   // dense scale table (+64 B: the padding lanes of a last partial block read past the last row)
        const size_t entries = (size_t)v.groups * v.N, wbytes = entries * (is_gptq ? 4 : 2) + 128;
        if (cudaMalloc(&m->wtab, wbytes) != cudaSuccess) { set_error("CUDA out of memory (scale table)"); cudaFree(m->tables); return fail(-3); }
        cudaMemsetAsync(m->wtab, 0, wbytes, stream);
        scale_table_kernel<<<(unsigned)((entries + 255) / 256), 256, 0, stream>>>(v, m->wtab);
        g_launch_count++;
        e = cudaStreamSynchronize(stream);
        if (e != cudaSuccess) { set_error("scale table failed: %s", cudaGetErrorString(e)); cudaFree(m->tables); cudaFree(m->wtab); return fail(-1); }
    }
    *out = (exl2b_qmatrix_t)m;
    return 0;
}

namespace exl2b {
int qmatrix_chain_buffers(QMatrix* m, bool wide) {
    half*& xp = wide ? m->xp_wide : m->xp_buf;
    float*& sq = wide ? m->sumsq_wide : m->sumsq_buf;
    if (xp) return 0;
    EXL2B_CUDA(cudaSetDevice(m->device));
    const size_t slots = wide ? 64 : 8;      // token slots of the layout: the widest tile of the row range
    const size_t xp_bytes = (size_t)m->v.K * 2 * slots, sq_bytes = ((size_t)m->v.K / 128 + 2) * slots * sizeof(float);
    EXL2B_CUDA(cudaMalloc(&xp, xp_bytes));
    EXL2B_CUDA(cudaMalloc(&sq, sq_bytes));
    EXL2B_CUDA(cudaMemset(xp, 0, xp_bytes));
    EXL2B_CUDA(cudaMemset(sq, 0, sq_bytes));
    return 0;
}
}  // namespace exl2b

extern "C" int exl2b_qmatrix_destroy(exl2b_qmatrix_t h) {
    QMatrix* m = (QMatrix*)h;
    if (!m) return 0;
    cudaSetDevice(m->device);
    if (m->tables) cudaFree(m->tables);
    if (m->owned_packed) cudaFree(m->owned_packed);
    if (m->wtab) cudaFree(m->wtab);
    if (m->xp_buf) cudaFree(m->xp_buf);
    if (m->sumsq_buf) cudaFree(m->sumsq_buf);
    if (m->xp_wide) cudaFree(m->xp_wide);
    if (m->sumsq_wide) cudaFree(m->sumsq_wide);
    delete m;
    return 0;
}

extern "C" int exl2b_qmatrix_info(exl2b_qmatrix_t h, int* height, int* width, int* groups, int* is_gptq,
                                  uint64_t* packed_bytes) {
    QMatrix* m = (QMatrix*)h;
    EXL2B_REQUIRE(m, "null handle");
    if (height) *height = m->v.K;
    if (width) *width = m->v.N;
    if (groups) *groups = m->v.groups;
    if (is_gptq) *is_gptq = m->v.is_gptq;
    if (packed_bytes) *packed_bytes = m->packed_bytes;
    return 0;
}

namespace exl2b {
// columns [strip0 * strip_n, (strip0 + nstrips) * strip_n) of the dequantised matrix into out[K, ld] (original row order)
int reconstruct_window(const QMatrix* m, half* out, int ld, int strip0, int nstrips, cudaStream_t stream) {
    dim3 grid(m->v.KS, nstrips), block(32 * strip_blocks(m->v.layout));
    reconstruct_kernel<<<grid, block, 0, stream>>>(m->v, 0, out, ld, strip0 * strip_n(m->v.layout), strip0);
    g_launch_count++;
    EXL2B_CUDA(cudaGetLastError());
    return 0;
}
}  // namespace exl2b

extern "C" int exl2b_reconstruct(exl2b_qmatrix_t h, uint16_t* out, exl2b_stream_t stream) {
    QMatrix* m = (QMatrix*)h;
    EXL2B_REQUIRE(m && out, "null argument");
    EXL2B_CUDA(cudaSetDevice(m->device));
    int gs = 0;
    dim3 grid(m->v.KS, m->v.strips), block(32 * strip_blocks(m->v.layout));
    reconstruct_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(m->v, gs, (half*)out, m->v.N, 0, 0);
    g_launch_count++;
    EXL2B_CUDA(cudaGetLastError());
    return 0;
}
