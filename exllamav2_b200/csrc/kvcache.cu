// Q4 / Q6 / Q8 K/V cache pack / unpack (exllamav2_ext/cuda/cache_q.cuh, cuda/cache.cu:143-497).
//
// Same arithmetic as the reference, op for op (so results are bit-identical to it on the same inputs):
//   pack:   Hadamard-32 and quantisation as kv_format.cuh defines them (the op order is stated there)
//   unpack: (q - 8) * scale (or (q - 128) * scale) -> Hadamard -> * 1/32
// wbits = 4: keys and values in 4 bits; 6: keys in 8 bits, values in 4 bits; 8: both in 8 bits (cache.cu:250-276).
// What differs is the mapping to the machine: the reference runs 256-thread CTAs over 512-value blocks staged
// through shared memory and, for the paged form, a (pages, 256, 2*batch) grid of mostly-empty CTAs
// (cache.cu:244-248).  The math is per 64-value warp unit, so here every warp independently converts 64-value
// units with direct coalesced global access (128 B in / 32 B + 4 B out per unit), the unit list is flattened
// over (k|v, sequence, token range) and the grid is sized to the actual work.
#include <algorithm>

#include "kv_format.cuh"

namespace exl2b {

// one warp: 64 fp16 values at `in` -> 64 * BITS / 8 packed bytes at `out`, 2 scales at `scales` (cache_q.cuh:78-108)
template <int BITS>
__device__ __forceinline__ void pack_unit(const half* __restrict__ in, uint8_t* __restrict__ out, half* __restrict__ scales,
                                          int lane) {
    constexpr int LPW = 16 / BITS;      // lanes per 32-bit output word
    const KvCodes c = kv_quantise<BITS>(hadamard32_h(reinterpret_cast<const half2*>(in)[lane], lane));
    uint32_t q = c.q0 | (c.q1 << BITS);
#pragma unroll
    for (int s = 1; s < LPW; s <<= 1) q |= (__shfl_down_sync(0xffffffffu, q, s) << (2 * BITS * s));
    if ((lane & (LPW - 1)) == 0) reinterpret_cast<uint32_t*>(out)[lane / LPW] = q;
    if ((lane & 15) == 0) scales[lane >> 4] = c.scale;
}

template <int BITS>
__device__ __forceinline__ void unpack_unit(const uint8_t* __restrict__ in, const half* __restrict__ scales,
                                            half* __restrict__ out, int lane) {
    constexpr int LPW = 16 / BITS, MASK = (1 << BITS) - 1, ZERO = 1 << (BITS - 1);
    const half scale = __ldg(scales + (lane >> 4));
    const uint32_t q = __ldg(reinterpret_cast<const uint32_t*>(in) + lane / LPW);
    const int shift0 = (lane & (LPW - 1)) * 2 * BITS;
    const int q0 = ((int)((q >> shift0) & MASK)) - ZERO;
    const int q1 = ((int)((q >> (shift0 + BITS)) & MASK)) - ZERO;
    half2 w2 = __halves2half2(__int2half_rn(q0), __int2half_rn(q1));
    w2 = __hmul2(w2, __half2half2(scale));
    w2 = hadamard32_h(w2, lane);
    w2 = __hmul2(w2, __float2half2_rn(1.0f / 32.0f));
    __stcg(reinterpret_cast<half2*>(out) + lane, w2);
}

struct KvJob {
    const void* k_a; void* k_b; void* k_s;     // pack: fp16 in, u8 out, scales out;  unpack: u8 in, fp16 out, scales in
    const void* v_a; void* v_b; void* v_s;
    int batch, dim, seq_stride;                // non-paged
    int offset_el, width_el;                   // non-paged element range per batch row (multiples of 64)
    int page_size, pages_per_seq, q_len;       // paged
    const int32_t* cache_seqlens;
    const int32_t* block_table;
    int units_per_seq;                         // upper bound of 64-value units per (k|v, sequence)
    int pack;
    int k_bits, v_bits;                        // element width of the quantised keys / values: 4 or 8
};

// Resolve unit index -> element offset.  Returns false when the unit is outside the sequence's live range.
__device__ __forceinline__ bool kv_unit_offset(const KvJob& J, int seq, int unit, size_t& el) {
    if (J.page_size == 0) {
        const int e = J.offset_el + unit * 64;
        if (e >= J.offset_el + J.width_el) return false;
        el = (size_t)seq * J.seq_stride + e;
        return true;
    }
    // paged: token range [a, b) of this sequence, widened to whole 512-value blocks like the reference
    // (cache.cu:177-184 pack, :350-357 unpack) when dim is not a multiple of 512
    const int seqlen = J.cache_seqlens[seq];
    int a, b;
    if (J.pack) { a = seqlen; b = seqlen + J.q_len; }
    else { if (!seqlen) return false; a = 0; b = seqlen; }
    long ea = (long)a * J.dim, eb = (long)b * J.dim;
    if (J.dim % 512) { ea = ea / 512 * 512; eb = (eb + 511) / 512 * 512; }
    const long e = ea + (long)unit * 64;
    if (e >= eb) return false;
    const long tok = e / J.dim;
    const int page_idx = (int)(tok / J.page_size);
    if (page_idx >= J.pages_per_seq) return false;
    const int page = J.block_table[(size_t)seq * J.pages_per_seq + page_idx];
    el = ((size_t)page * J.page_size + (size_t)(tok - (long)page_idx * J.page_size)) * J.dim + (size_t)(e - tok * J.dim);
    return true;
}

__global__ void __launch_bounds__(256) kv_q_kernel(const __grid_constant__ KvJob J) {
    griddep_launch_dependents();
    griddep_wait();
    const int lane = threadIdx.x & 31;
    const long per_kv = (long)J.batch * J.units_per_seq;
    const int nkv = J.v_a ? 2 : 1;
    const long total = per_kv * nkv;
    const long nwarps = ((long)gridDim.x * blockDim.x) >> 5;
    // grid-stride over 64-value units: the grid is capped at a few CTAs per SM, dead units cost one compare
    for (long wid = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; wid < total; wid += nwarps) {
        const int kv = (int)(wid / per_kv);
        const long r = wid - (long)kv * per_kv;
        const int seq = (int)(r / J.units_per_seq), unit = (int)(r - (long)seq * J.units_per_seq);
        size_t el;
        if (!kv_unit_offset(J, seq, unit, el)) continue;
        const void* a = kv ? J.v_a : J.k_a;
        void* b = kv ? J.v_b : J.k_b;
        void* s = kv ? J.v_s : J.k_s;
        const bool q8 = (kv ? J.v_bits : J.k_bits) == 8;      // warp-uniform
        if (J.pack) {
            if (q8) pack_unit<8>((const half*)a + el, (uint8_t*)b + el, (half*)s + el / 32, lane);
            else pack_unit<4>((const half*)a + el, (uint8_t*)b + el / 2, (half*)s + el / 32, lane);
        } else {
            if (q8) unpack_unit<8>((const uint8_t*)a + el, (const half*)s + el / 32, (half*)b + el, lane);
            else unpack_unit<4>((const uint8_t*)a + el / 2, (const half*)s + el / 32, (half*)b + el, lane);
        }
    }
}

static int kv_launch(KvJob& J, cudaStream_t stream) {
    const long warps = (long)J.batch * J.units_per_seq * (J.v_a ? 2 : 1);
    if (warps <= 0) return 0;
    int dev = 0;
    cudaGetDevice(&dev);
    const long cap = (long)device_sm_count(dev) * 8;
    const long blocks = std::min((warps + 7) / 8, cap);
    EXL2B_CUDA(launch_pdl(kv_q_kernel, dim3((unsigned)blocks), dim3(256), 0, stream, J));
    return 0;
}

static int kv_common(KvJob& J, int batch, int dim, int seq_stride, int offset, int width, int page_size,
                     const int32_t* cache_seqlens, const int32_t* block_table, int pages_per_seq, int wbits) {
    EXL2B_REQUIRE(wbits == 4 || wbits == 6 || wbits == 8, "cache wbits must be 4 (Q4), 6 (Q6) or 8 (Q8); got %d", wbits);
    J.k_bits = wbits == 4 ? 4 : 8;
    J.v_bits = wbits == 8 ? 8 : 4;
    EXL2B_REQUIRE(dim > 0 && dim % 64 == 0, "kv dim %d must be a multiple of 64", dim);
    J.batch = batch;
    J.dim = dim;
    J.seq_stride = seq_stride;
    J.page_size = page_size;
    J.pages_per_seq = pages_per_seq;
    J.cache_seqlens = cache_seqlens;
    J.block_table = block_table;
    if (page_size == 0) {
        EXL2B_REQUIRE(seq_stride % dim == 0 && offset >= 0 && width >= 0 && (long)(offset + width) * dim <= seq_stride,
                      "tokens [%d, %d) outside the %d tokens of a batch row", offset, offset + width, seq_stride / dim);
        // ext_cache.cpp:150-157: widen [offset, offset+width) tokens to 512-element block boundaries -- but not past the end of
        // the batch row (seq_stride): beyond it lie the next row's tokens and, after the last row, no tensor at all
        if (dim % 512) {
            while (((long)offset * dim) % 512) offset--;
            while (((long)width * dim) % 512) width++;
        }
        J.offset_el = offset * dim;
        J.width_el = (int)std::min((long)width * dim, (long)seq_stride - J.offset_el);
        J.units_per_seq = J.width_el / 64;
    } else {
        EXL2B_REQUIRE(cache_seqlens && block_table && pages_per_seq > 0, "paged kv needs cache_seqlens and block_table");
        J.q_len = width;
        const long tokens = J.pack ? (long)width : (long)pages_per_seq * page_size;
        J.units_per_seq = (int)((tokens * dim + 511) / 512 * 8 + 8);
    }
    return 0;
}

}  // namespace exl2b

using namespace exl2b;

extern "C" int exl2b_fp16_to_q_kv(const uint16_t* k_in, uint8_t* k_out, uint16_t* k_scales, const uint16_t* v_in,
                                  uint8_t* v_out, uint16_t* v_scales, int batch, int dim, int seq_stride, int offset,
                                  int width, int page_size, const int32_t* cache_seqlens, const int32_t* block_table,
                                  int pages_per_seq, int wbits, exl2b_stream_t stream) {
    EXL2B_REQUIRE(k_in && k_out && k_scales, "null k tensors");
    KvJob J = {};
    J.pack = 1;
    J.k_a = k_in; J.k_b = k_out; J.k_s = k_scales;
    J.v_a = v_in; J.v_b = v_out; J.v_s = v_scales;
    int rc = kv_common(J, batch, dim, seq_stride, offset, width, page_size, cache_seqlens, block_table, pages_per_seq, wbits);
    if (rc) return rc;
    return kv_launch(J, (cudaStream_t)stream);
}

extern "C" int exl2b_q_to_fp16_kv(const uint8_t* k_in, const uint16_t* k_scales, uint16_t* k_out, const uint8_t* v_in,
                                  const uint16_t* v_scales, uint16_t* v_out, int batch, int dim, int seq_stride,
                                  int offset, int width, int page_size, const int32_t* cache_seqlens,
                                  const int32_t* block_table, int pages_per_seq, int wbits, exl2b_stream_t stream) {
    EXL2B_REQUIRE(k_in && k_out && k_scales, "null k tensors");
    KvJob J = {};
    J.pack = 0;
    J.k_a = k_in; J.k_b = k_out; J.k_s = (void*)k_scales;
    J.v_a = v_in; J.v_b = v_out; J.v_s = (void*)v_scales;
    int rc = kv_common(J, batch, dim, seq_stride, offset, width, page_size, cache_seqlens, block_table, pages_per_seq, wbits);
    if (rc) return rc;
    return kv_launch(J, (cudaStream_t)stream);
}
