// Private HBM layout of a quantized matrix and the register-level unpack -- shared by the repack kernel, the GEMV / GEMM
// kernels, reconstruct, and the host-side emulation in tests/emu (compiled with g++).
//
// The reference keeps the checkpoint's [packed-row, column] order and re-shuffles bit fields inside each 32-row column unit at
// load time (exllamav2_ext/cuda/q_matrix.cu:21-44, quant/qdq_*.cuh shuffle_*).  We do a different load-time re-pack (same
// total bytes, written back over q_weight exactly like the reference mutates it) into a layout built for streaming with TMA bulk copies.
//
// THE layout every kernel uses (LAYOUT_TC below):
//   strip  = 128 output columns = 4 blocks; block = 32 k x 32 n; every block's slabs (32 stored rows k' each) form their own
//            contiguous byte stream over K: [strip][block][slab].  Any (block, k-range) is ONE contiguous byte range that a
//            warp fetches with cp.async.bulk (TMA 1-D).  Mixed bit widths along K only change the slab stride of a region.
//   lane l of a block owns column n = l and all 32 k of the slab: value i <-> k_local = i, pair p = i / 2 = (k, k+1).
//   plane  = a b-bit value is split into power-of-two bit planes (b = main + extra: 2=2, 3=2+1, 4=4, 5=4+1, 6=4+2, 8=8) with
//            field e of pair slot j at bit 16e + P*j of its word, so that
//              * `(w >> sh) & mask | magic` is a valid fp16 pair (the 0x6400 trick generalised to every exponent): the wgmma
//                kernel stores it straight into row n of its shared-memory A tile (gemm_tc.cu);
//              * `w & 0x0f0f0f0f` / `w & 0xf0f0f0f0` (and the 2- / 1-bit analogues) are four BYTE operands of the integer
//                dot-product instruction: the batch-1 GEMV feeds packed words to dp4a unexpanded (gemv_i8.cu).
//
// The round-1 mma.sync fragment layout (LAYOUT_MMA: strip = 64 columns, lane (g, t) owns n in {g, g+8, g+16, g+24} and
// k in {8t..8t+7}) is no longer produced by the library; its index algebra stays here because tests/emu checks the
// compose / extract / unpack logic for both mappings.
//   Value index inside a lane's 32 values (MMA mapping):  i = p*2 + e,  pair p = sub*8 + s*4 + reg,  reg = h*2 + rr
//   n_local = sub*16 + rr*8 + g,  k_local = 8t + 4s + 2h + e
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define EXL2B_HD __host__ __device__ __forceinline__
#else
#define EXL2B_HD inline
#endif

namespace exl2b {

constexpr int SLAB_K = 32;
constexpr int BLOCK_N = 32;
constexpr int STRIP_BLOCKS = 2;
constexpr int STRIP_N = BLOCK_N * STRIP_BLOCKS;   // 64

EXL2B_HD constexpr int plane_main(int bits) { return bits == 2 ? 2 : bits == 3 ? 2 : bits == 8 ? 8 : 4; }
EXL2B_HD constexpr int plane_extra(int bits) { return bits == 3 ? 1 : bits == 5 ? 1 : bits == 6 ? 2 : 0; }
EXL2B_HD constexpr bool bits_supported(int b) { return b == 2 || b == 3 || b == 4 || b == 5 || b == 6 || b == 8; }

// bytes of one block / one slab at a bit width (== the checkpoint's bytes for the same values)
EXL2B_HD constexpr int block_bytes(int bits) { return 128 * bits; }
EXL2B_HD constexpr int slab_bytes(int bits) { return block_bytes(bits) * STRIP_BLOCKS; }

// A plane with P bits per field stores P words per lane (32 values * P bits).  Segment = lane-major array of
// up to 4 words per lane (so a lane's words are one aligned 4/8/16-byte shared-memory load); the 8-bit plane is
// two 4-word segments.  Word offsets (in uint32) of a segment inside a block:
EXL2B_HD constexpr int main_words(int bits) { return plane_main(bits); }          // words per lane
EXL2B_HD constexpr int extra_words(int bits) { return plane_extra(bits); }
// main plane: P<=4: one segment at word 0 with P words/lane. P==8: segment A (pairs 0..7) at 0, B at 128.
EXL2B_HD constexpr int main_seg_words(int bits) { return plane_main(bits) == 8 ? 4 : plane_main(bits); }
EXL2B_HD constexpr int extra_seg_base(int bits) { return 32 * plane_main(bits); }   // in words, from block start

// pair slot p (0..15) of a plane with P bits: which word of the lane, and field slot j inside the word
EXL2B_HD constexpr int pairs_per_word(int P) { return 16 / P; }
// The assignment pair -> (word, slot) is chosen per plane width so that every plane presents the SAME byte order to the integer
// dot product: masking field position i of word w of ANY plane leaves the four bytes (k0, k0+4, k0+1, k0+5) of one 8-k octet
// half (k0 = 8*(m>>1) + 2*(m&1) for operand word m), i.e. pairs p0 = 4*(m>>1) + (m&1) and p0 + 2.  The batch-1 GEMV stages the
// row ONCE in that order and never permutes an operand (gemv_i8.cu):
//   P = 4: word w, low / high nibbles  <-> m = 2w, 2w+1          (pairs 4w, 4w+2 | 4w+1, 4w+3)
//   P = 2: word w, field position i    <-> m = 4w + i            P = 1: bit position i <-> m = i        P = 8: word w <-> m = w
EXL2B_HD constexpr int pair_word(int P, int p) {
    return P == 4 ? p / 4 : P == 2 ? (p >> 3) : P == 1 ? 0 : /* P == 8 */ 2 * (p >> 2) + (p & 1);
}
EXL2B_HD constexpr int pair_slot(int P, int p) {
    return P == 4 ? p % 4
         : P == 2 ? 4 * ((p >> 1) & 1) + 2 * ((p & 7) >> 2) + (p & 1)
         : P == 1 ? 8 * ((p >> 1) & 1) + 2 * (p >> 2) + (p & 1)
         : /* P == 8 */ (p >> 1) & 1;
}
// field e of pair slot j sits at bit  16*e + P*j  of its word
EXL2B_HD constexpr int field_bit(int P, int j, int e) { return 16 * e + P * j; }
// extraction: shift the word right by sh, then the field is at in-halfword offset off (off + P <= 10)
EXL2B_HD constexpr int field_sh(int P, int j) { return (P * j + P <= 10) ? 0 : ((P == 4 || P == 8) ? 8 : 10); }
EXL2B_HD constexpr int field_off(int P, int j) { return P * j - field_sh(P, j); }
EXL2B_HD constexpr uint32_t field_mask(int P, int j) {
    return (uint32_t)(((1u << P) - 1u) << field_off(P, j)) * 0x00010001u;
}
// fp16 magic: exponent E = 10 - off so that  bits(mask&w | magic)  ==  2^E + field   exactly
EXL2B_HD constexpr int field_exp(int P, int j) { return 10 - field_off(P, j); }
EXL2B_HD constexpr uint32_t field_magic(int P, int j) { return (uint32_t)((field_exp(P, j) + 15) << 10) * 0x00010001u; }

// fp16 bit pattern of a (possibly negative) integer-valued constant that is exactly representable
EXL2B_HD constexpr uint16_t f16_bits_of_int(int v) {
    // v = +-m * 2^k with m < 2048
    if (v == 0) return 0;
    uint16_t sign = v < 0 ? 0x8000 : 0;
    uint32_t a = (uint32_t)(v < 0 ? -v : v);
    int e = 0;
    while ((a >> e) >= 2048u) e++;          // drop low zero bits (caller guarantees exactness)
    uint32_t m = a >> e;
    int top = 0;
    while ((m >> (top + 1)) != 0) top++;    // position of leading one
    int exp = top + e;                      // value = 1.xxx * 2^exp
    uint32_t frac = ((m << (10 - top)) & 0x3FFu);
    return (uint16_t)(sign | ((uint32_t)(exp + 15) << 10) | frac);
}
EXL2B_HD constexpr uint32_t h2_const_int(int v) { return (uint32_t)f16_bits_of_int(v) * 0x00010001u; }

// --------------------------------------------------------------------------------------------------------------
// where a value lives (used by the repack kernel and the host emulation)
// --------------------------------------------------------------------------------------------------------------
struct ValuePos { int n_local; int k_local; };
EXL2B_HD constexpr ValuePos value_pos(int lane, int i) {
    int g = lane >> 2, t = lane & 3;
    int e = i & 1, p = i >> 1;
    int rr = p & 1, h = (p >> 1) & 1, s = (p >> 2) & 1, sub = (p >> 3) & 1;
    return ValuePos{sub * 16 + rr * 8 + g, 8 * t + 4 * s + 2 * h + e};
}
// inverse: which (lane, i) holds (n_local, k_local)
EXL2B_HD constexpr int lane_of(int n_local, int k_local) { return ((n_local & 7) << 2) | (k_local >> 3); }
EXL2B_HD constexpr int index_of(int n_local, int k_local) {
    int sub = n_local >> 4, rr = (n_local >> 3) & 1;
    int kk = k_local & 7;
    int s = kk >> 2, h = (kk >> 1) & 1, e = kk & 1;
    int p = sub * 8 + s * 4 + h * 2 + rr;
    return p * 2 + e;
}

// ---- second lane mapping ("TC" layout, used by the wgmma kernel) ------------------------------------------------------
// strip = 128 columns = 4 blocks; each block's slabs form their own contiguous stream ([strip][blk][slab]), lane l of a
// block owns column n = l and all 32 k of the slab: value i <-> k_local = i, pair p = i/2 = (k, k+1).  After unpacking,
// register p of lane l is half2(W[k=2p][n], W[2p+1][n]) -- four registers are one 16-byte core-matrix row (8 k) of row n of
// the wgmma A operand (M = 128 weight columns, no-swizzle K-major tile in shared memory).
constexpr int LAYOUT_MMA = 0;   // mma.sync fragment layout above (strip 64)
constexpr int LAYOUT_TC = 1;    // column-per-lane row layout (strip 128)
EXL2B_HD constexpr int strip_n(int layout) { return layout == LAYOUT_TC ? 128 : 64; }
EXL2B_HD constexpr int strip_blocks(int layout) { return layout == LAYOUT_TC ? 4 : 2; }
EXL2B_HD constexpr ValuePos value_pos_l(int layout, int lane, int i) {
    return layout == LAYOUT_TC ? ValuePos{lane, i} : value_pos(lane, i);
}

// Compose the lane's plane words from its 32 integer values q[i] (0 <= q < 2^bits).
// out_main: main_words(bits) words, out_extra: extra_words(bits) words.
EXL2B_HD void compose_lane_words(int bits, const uint32_t* q, uint32_t* out_main, uint32_t* out_extra) {
    const int Pm = plane_main(bits), Pe = plane_extra(bits);
    for (int w = 0; w < Pm; ++w) out_main[w] = 0u;
    for (int w = 0; w < Pe; ++w) out_extra[w] = 0u;
    for (int i = 0; i < 32; ++i) {
        int p = i >> 1, e = i & 1;
        uint32_t fm = q[i] & ((1u << Pm) - 1u);
        out_main[pair_word(Pm, p)] |= fm << field_bit(Pm, pair_slot(Pm, p), e);
        if (Pe) {
            uint32_t fe = (q[i] >> Pm) & ((1u << Pe) - 1u);
            out_extra[pair_word(Pe, p)] |= fe << field_bit(Pe, pair_slot(Pe, p), e);
        }
    }
}

// word offset (uint32 units, from the block start) of word `w` of lane `lane` in the main / extra plane
EXL2B_HD constexpr int main_word_index(int bits, int lane, int w) {
    return plane_main(bits) == 8 ? ((w >> 2) * 128 + lane * 4 + (w & 3)) : (lane * plane_main(bits) + w);
}
EXL2B_HD constexpr int extra_word_index(int bits, int lane, int w) {
    return extra_seg_base(bits) + lane * plane_extra(bits) + w;
}

// Inverse of compose (integer domain; the fp16-domain unpack used by the kernels is in dequant.cuh).
EXL2B_HD uint32_t extract_value(int bits, const uint32_t* lane_main, const uint32_t* lane_extra, int i) {
    const int Pm = plane_main(bits), Pe = plane_extra(bits);
    int p = i >> 1, e = i & 1;
    uint32_t v = (lane_main[pair_word(Pm, p)] >> field_bit(Pm, pair_slot(Pm, p), e)) & ((1u << Pm) - 1u);
    if (Pe) v |= ((lane_extra[pair_word(Pe, p)] >> field_bit(Pe, pair_slot(Pe, p), e)) & ((1u << Pe) - 1u)) << Pm;
    return v;
}

}  // namespace exl2b
