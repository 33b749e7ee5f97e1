// fp16-domain unpack of one lane's 32 values of a block into mma.m16n8k16 A-fragments (see layout.h).
// Replaces the reference's dequant_{2,3,4,5,6,8}bit_* (exllamav2_ext/cuda/quant/qdq_*.cuh): same idea
// ("(q & mask) | magic" is already an fp16), generalised so that every field of every bit width is one
// LOP3 + one HADD2 (single-plane widths) or two LOP3 + HFMA2 + HADD2 (3/5/6-bit), all EXACT in fp16
// (every intermediate is an integer of magnitude < 2048, or a power-of-two multiple with <= 11 significant bits).
//
// Compiles for device (real half2 intrinsics) and for host (bit-exact emulation with _Float16) so that
// tests/emu can run the very same index/constant logic on the CPU.
#pragma once
#include "layout.h"

#if defined(__CUDA_ARCH__)
#include <cuda_fp16.h>
namespace exl2b {
__device__ __forceinline__ uint32_t h2add_bits(uint32_t a, uint32_t b) {
    uint32_t r;
    asm("add.rn.f16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
__device__ __forceinline__ uint32_t h2fma_bits(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t r;
    asm("fma.rn.f16x2 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}
__device__ __forceinline__ uint32_t h2mul_bits(uint32_t a, uint32_t b) {
    uint32_t r;
    asm("mul.rn.f16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
// (x & mask) | magic as ONE LOP3 (the compiler otherwise emits AND + OR when both constants are immediates)
__device__ __forceinline__ uint32_t and_or(uint32_t x, uint32_t mask, uint32_t magic) {
    uint32_t r;
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(r) : "r"(x), "r"(mask), "r"(magic));
    return r;
}
}  // namespace exl2b
#else
#include <string.h>
namespace exl2b {
static inline double h_to_d(uint16_t h) { _Float16 x; memcpy(&x, &h, 2); return (double)x; }
static inline uint16_t d_to_h(double d) { _Float16 x = (_Float16)d; uint16_t h; memcpy(&h, &x, 2); return h; }
static inline uint32_t h2add_bits(uint32_t a, uint32_t b) {
    uint32_t lo = d_to_h(h_to_d((uint16_t)a) + h_to_d((uint16_t)b));
    uint32_t hi = d_to_h(h_to_d((uint16_t)(a >> 16)) + h_to_d((uint16_t)(b >> 16)));
    return lo | (hi << 16);
}
static inline uint32_t h2fma_bits(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t lo = d_to_h(h_to_d((uint16_t)a) * h_to_d((uint16_t)b) + h_to_d((uint16_t)c));
    uint32_t hi = d_to_h(h_to_d((uint16_t)(a >> 16)) * h_to_d((uint16_t)(b >> 16)) + h_to_d((uint16_t)(c >> 16)));
    return lo | (hi << 16);
}
static inline uint32_t h2mul_bits(uint32_t a, uint32_t b) {
    uint32_t lo = d_to_h(h_to_d((uint16_t)a) * h_to_d((uint16_t)b));
    uint32_t hi = d_to_h(h_to_d((uint16_t)(a >> 16)) * h_to_d((uint16_t)(b >> 16)));
    return lo | (hi << 16);
}
static inline uint32_t and_or(uint32_t x, uint32_t mask, uint32_t magic) { return (x & mask) | magic; }
}  // namespace exl2b
#endif

namespace exl2b {

// constants of pair p
template <int BITS> struct PairConst {
    static constexpr int Pm = plane_main(BITS);
    static constexpr int Pe = plane_extra(BITS);
    static constexpr int zp = 1 << (BITS - 1);
    EXL2B_HD static constexpr int em(int p) { return field_exp(Pm, pair_slot(Pm, p)); }
    EXL2B_HD static constexpr int ee(int p) { return Pe ? field_exp(Pe, pair_slot(Pe ? Pe : 1, p)) : 0; }
    // single plane:  v = t + c1,  c1 = -(2^Em + zp)
    EXL2B_HD static constexpr int c_single(int p, int zero) { return -((1 << em(p)) + zero); }
    // two planes:    r1 = te * 2^Pm + k1,   k1 = -(2^(Pm+Ee) + 2^Em + zp);   v = tm + r1
    EXL2B_HD static constexpr int k_double(int p, int zero) { return -((1 << (Pm + ee(p))) + (1 << em(p)) + zero); }
};

// Unpack the lane's 32 values into A[16] (A[p] = half2 bits of pair p, value = q - zero).
//   mw: main-plane words (plane_main(BITS) of them), ew: extra-plane words (plane_extra(BITS) of them).
// EXL2: zero = 2^(BITS-1) for every value (symmetric zero point, qdq_4.cuh:34-60 etc.).
template <int BITS>
EXL2B_HD void dequant_block_exl2(const uint32_t* mw, const uint32_t* ew, uint32_t* A) {
    using PC = PairConst<BITS>;
    constexpr int Pm = PC::Pm, Pe = PC::Pe;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int p = 0; p < 16; ++p) {
        const int jm = pair_slot(Pm, p);
        const uint32_t x = mw[pair_word(Pm, p)] >> field_sh(Pm, jm);
        const uint32_t tm = and_or(x, field_mask(Pm, jm), field_magic(Pm, jm));
        if (Pe == 0) {
            A[p] = h2add_bits(tm, h2_const_int(PC::c_single(p, PC::zp)));
        } else {
            const int PeS = Pe ? Pe : 1;
            const int je = pair_slot(PeS, p);
            const uint32_t y = ew[pair_word(PeS, p)] >> field_sh(PeS, je);
            const uint32_t te = and_or(y, field_mask(PeS, je), field_magic(PeS, je));
            const uint32_t r1 = h2fma_bits(te, h2_const_int(1 << Pm), h2_const_int(PC::k_double(p, PC::zp)));
            A[p] = h2add_bits(tm, r1);
        }
    }
}

// GPTQ 4-bit: per-row zero point (z+1), cuda/q_gemm_kernel_gptq.cuh:167-172.  In the 4-bit plane the field
// exponent depends only on rr = p & 1 (E = 10 for rr = 0, 6 for rr = 1), so four constants cover the block:
//   zc[sub*2 + rr] = half2 bits of -(2^E + z + 1) for row n_local = sub*16 + rr*8 + g.
EXL2B_HD uint32_t gptq_zero_const(int rr, int zero_plus_1) {
    const int E = rr ? 6 : 10;
    return h2_const_int(-((1 << E) + zero_plus_1));
}
EXL2B_HD void dequant_block_gptq(const uint32_t* mw, const uint32_t* zc, uint32_t* A) {
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int p = 0; p < 16; ++p) {
        const int jm = pair_slot(4, p);
        const uint32_t x = mw[pair_word(4, p)] >> field_sh(4, jm);
        const uint32_t tm = and_or(x, field_mask(4, jm), field_magic(4, jm));
        A[p] = h2add_bits(tm, zc[((p >> 3) & 1) * 2 + (p & 1)]);
    }
}

// 4-bit fast path ("offset form"): every nibble is moved to in-halfword offset 4 so ONE mask / ONE magic serve all
// fields and the zero point is not subtracted per weight:  A[p] = half2(64 + q).  The GEMV removes the offset per
// group with the activation sum that an extra all-ones mma row provides:  sum a*(q - z) = sum a*(64+q) - (64+z)*sum a.
// 3 shifts + 4 LOP3 per 8 weights (vs 1 shift + 4 LOP3 + 4 HADD2).  Exact: 64+q is an fp16 integer, products are
// exact in the tensor core, fp32 accumulation sees operands only 16x larger than q - z.
constexpr int OFFSET4 = 64;
EXL2B_HD void dequant_block_4bit_offset(const uint32_t* mw, uint32_t* A) {
    const uint32_t mask = 0x00f000f0u, magic = 0x54005400u;      // fp16 64.0 | nibble at mantissa bits 4..7 = 64 + q
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int w = 0; w < 4; ++w) {           // word w = (sub, s); slots 0..3 = mma regs 0..3
        const uint32_t x = mw[w];
        A[w * 4 + 0] = and_or(x << 4, mask, magic);
        A[w * 4 + 1] = and_or(x, mask, magic);
        A[w * 4 + 2] = and_or(x >> 4, mask, magic);
        A[w * 4 + 3] = and_or(x >> 8, mask, magic);
    }
}

// Two-offset form: no shift for slots 0/1, one shift for slots 2/3 -> 4 LOP3 + 1 SHF per 8 weights, all on the ALU pipe,
// which is what bounds the unpack.
//   even pair slots: (x & 0x000f000f) | 0x6400 = 1024 + q      odd pair slots: (x & 0x00f000f0) | 0x5400 = 64 + q
// The per-slot offset (+ the zero point) is removed by one extra MMA against a constant "offset tile".
EXL2B_HD constexpr int offset2_of_pair(int p) { return (p & 1) ? 64 : 1024; }
EXL2B_HD void dequant_block_4bit_offset2(const uint32_t* mw, uint32_t* A) {
    const uint32_t m0 = 0x000f000fu, g0 = 0x64006400u, m1 = 0x00f000f0u, g1 = 0x54005400u;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int w = 0; w < 4; ++w) {
        const uint32_t x = mw[w], y = x >> 8;
        A[w * 4 + 0] = and_or(x, m0, g0);
        A[w * 4 + 1] = and_or(x, m1, g1);
        A[w * 4 + 2] = and_or(y, m0, g0);
        A[w * 4 + 3] = and_or(y, m1, g1);
    }
}

}  // namespace exl2b
