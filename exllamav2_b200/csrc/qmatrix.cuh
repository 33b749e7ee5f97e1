// Internal QMatrix handle (the reference's class QMatrix, exllamav2_ext/cuda/q_matrix.cuh:11-83).
#pragma once
#include <vector>

#include "common.cuh"

namespace exl2b {

// A run of slabs with one bit width and one (power-of-two) group size: everything about slab ks in the region is
// arithmetic on kernel parameters -- no table load sits on the GEMV's critical path.
struct QRegion {
    int ks_begin;        // first slab of the region (the region ends where the next one begins, or at KS)
    int bits;
    int spg_log2;        // log2(slabs per group)
    int group_base;      // group index of the region's first slab
    uint32_t off_base;   // byte offset of the region's first slab inside a strip
};
constexpr int MAX_REGIONS = 6;

// Device-side view handed to kernels by value.
struct QMatView {
    const uint32_t* packed;       // [strips][strip_bytes]  private layout
    const uint2* slab_tab;        // [KS]  .x = byte offset of the slab inside a strip (MMA) / inside a block stream (TC),
                                  //       .y = group | bits << 16 | slabs-left-with-same-bits << 20
    const uint32_t* q_scale;      // EXL2 int32[G, N/8]   (checkpoint layout, read directly)
    const half* q_scale_max;      // EXL2 fp16[G]
    const uint32_t* qzeros;       // GPTQ int32[G, N/8]
    const half* gptq_scales;      // GPTQ fp16[G, N]
    const uint16_t* perm;         // [K] or NULL
    const half* bias;             // [N] or NULL
    uint32_t strip_bytes;         // bytes of one strip (all blocks, all K)
    uint32_t blk_stream_bytes;    // LAYOUT_TC: bytes of one block's stream over K (strip_bytes / 4)
    int layout;                   // LAYOUT_MMA (strip 64, [strip][slab][blk]) or LAYOUT_TC (strip 128, [strip][blk][slab])
    int K, N, KS, strips, groups;
    int is_gptq;
    int num_regions;
    QRegion reg[MAX_REGIONS];
};

struct QMatrix {
    int device = 0;
    QMatView v = {};
    uint32_t* owned_packed = nullptr;   // only when width % 64 != 0 (padded copy); otherwise packed aliases q_weight
    void* tables = nullptr;             // slab_tab storage
    uint32_t bits_mask = 0;             // bit b set <=> some group uses b bits
    uint64_t packed_bytes = 0;
    std::vector<uint2> slab_tab_host;
    const uint16_t* invperm = nullptr;  // q_invperm of the checkpoint (device), NULL = identity
    void* wtab = nullptr;               // dense per-(group, column) scale table of the batch-1 GEMV (gemv_i8.cu): EXL2 fp16[G][N] =
                                        //   dq_scale(q_scale nibble, q_scale_max); GPTQ uint32[G][N] = fp16 scale | (qzero + 1) << 16
    half* xp_buf = nullptr;             // chained launches: this matrix's input, written by its producer's epilogue
    float* sumsq_buf = nullptr;         //   and the producer's per-strip sums of squares (deferred RMSNorm); 1..8 rows: K x 16 B
                                        //   (8 token slots), [strips][8]
    half* xp_wide = nullptr;            // the same for chained launches of 9..64 rows: K x 128 B (64 token slots), [strips][64]
    float* sumsq_wide = nullptr;
};
// allocate xp_buf / sumsq_buf (wide: xp_wide / sumsq_wide) on first use (never inside a stream capture: call once eagerly
// first).  Neither pair is ever moved or regrown: a graph captured over one stays valid when the other is created.
int qmatrix_chain_buffers(QMatrix* m, bool wide = false);

inline uint32_t meta_group(uint32_t m) { return m & 0xFFFFu; }
inline uint32_t meta_bits(uint32_t m) { return (m >> 16) & 0xFu; }
inline uint32_t meta_left(uint32_t m) { return m >> 20; }

}  // namespace exl2b
