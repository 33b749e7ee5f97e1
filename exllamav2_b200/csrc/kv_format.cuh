// The Q4 / Q6 / Q8 K/V cache format (exllamav2_ext/cuda/cache_q.cuh): one definition for the cache's pack / unpack
// kernels (kvcache.cu) and the fused decode attention that reads and appends the cache (attn_q4.cu).
//
// A 64-value unit of a head row is two interleaved 32-vectors (a warp holds elements 2 lane, 2 lane + 1 as one half2); each
// is rotated by the unnormalised Hadamard-32 butterfly and quantised with one fp16 scale per 32 consecutive rotated values.
// The op order is the reference's, so the stored bits match it exactly:
//   absmax over the 16 lanes of a 32-value block, w = w / absmax * Z + Z, q = clamp(rn(w), 0, 2Z - 1), scale = absmax / Z
// with Z = 8 at 4 bits (two values per byte, low nibble first) and Z = 128 at 8 bits (one value per byte).
#pragma once
#include "common.cuh"

namespace exl2b {

// fp16 Hadamard-32 across the warp on both halves of a half2 (fp16 adds, exact sign flips)
__device__ __forceinline__ half2 hadamard32_h(half2 w2, int lane) {
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

// the same butterfly in fp32 on both halves of a float2 (the attention kernel's query, new rows and output)
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

struct KvCodes {
    int q0, q1;       // codes of this lane's two values, 0 .. 2^BITS - 1
    half scale;       // scale of the lane's 32-value block
};

// quantise this lane's two values of a rotated unit (hadamard32_h output) to BITS = 4 or 8 bits
template <int BITS>
__device__ __forceinline__ KvCodes kv_quantise(half2 w2) {
    static_assert(BITS == 4 || BITS == 8, "cache elements are 4 or 8 bits");
    constexpr float Z = BITS == 4 ? 8.0f : 128.0f;
    constexpr int QMAX = (1 << BITS) - 1;
    const half2 absmax2 = __habs2(w2);
    half absmax = __hmax(__low2half(absmax2), __high2half(absmax2));
    absmax = __hmax(absmax, __shfl_xor_sync(0xffffffffu, absmax, 8));
    absmax = __hmax(absmax, __shfl_xor_sync(0xffffffffu, absmax, 4));
    absmax = __hmax(absmax, __shfl_xor_sync(0xffffffffu, absmax, 2));
    absmax = __hmax(absmax, __shfl_xor_sync(0xffffffffu, absmax, 1));
    const half2 cz = __half2half2(__float2half_rn(Z));
    w2 = __h2div(w2, __half2half2(absmax));
    w2 = __hfma2(w2, cz, cz);
    KvCodes c;
    c.q0 = min(max(__half2int_rn(__low2half(w2)), 0), QMAX);
    c.q1 = min(max(__half2int_rn(__high2half(w2)), 0), QMAX);
    c.scale = __hmul(absmax, __float2half_rn(1.0f / Z));
    return c;
}

}  // namespace exl2b
