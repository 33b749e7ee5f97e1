// Internal interface of the streaming dequant-GEMV (gemv.cu), shared with the fused attention / MLP blocks.
#pragma once
#include "qmatrix.cuh"

namespace exl2b {

constexpr int GEMV_MAX_MATS = 3;
constexpr int GEMV_MTOK = 8;          // tokens per pass (the N=8 dimension of wgmma.m64n8k16)
constexpr int GEMV_MAX_CHAIN_ROWS = 64;   // rows of one chained launch: the widest token tile (wgmma.m64n64k16), one pass
// token tile of a wgmma launch of `rows` rows in one pass: 8 (1..8 rows), 32 (9..32) or 64 (33..64)
constexpr int tc_tile(int rows) { return rows <= GEMV_MTOK ? GEMV_MTOK : rows <= 32 ? 32 : 64; }
// Per (device, stream) scratch of the wgmma kernel (gemv_workspace): the 8-row split-K workspace and activation scratch, and
// the wide tiles' own, created on the first launch of more than 8 rows with extras.  The activation scratch holds 3 matrices
// of K <= 65536 at 16 B (8 token slots) or 128 B (64) per k.  The wide workspace covers 64-row partials of a 152064-column head
// at two contributors per strip (stream-K over one CTA per SM).
constexpr size_t TC_WS_BYTES = (size_t)32 << 20;
constexpr size_t TC_WIDE_WS_BYTES = (size_t)96 << 20;
constexpr size_t TC_XP_BYTES = (size_t)GEMV_MAX_MATS * 65536 * 16;
constexpr size_t TC_WIDE_XP_BYTES = (size_t)GEMV_MAX_MATS * 65536 * 128;

enum GemvEpilogue : int {
    EPI_STORE = 0,      // c = (clear ? 0 : c) + bias + acc
    EPI_SILU_MUL = 1,   // mats = {gate, up}: c0 = silu(gate) * up   (written to mat[0].c only)
    EPI_GELU_MUL = 2,
};

struct GemvMat {
    QMatView w;
    const half* xp;  // wgmma path: activations prepared by tc_prep_kernel (normalised, permuted, core-matrix layout)
    const half* x;   // input activations fp16 [M][ldx], ORIGINAL feature order (the kernel gathers through w.perm)
    int ldx;
    half* c;         // output fp16 [M][ldc]
    int ldc;
    int clear;       // 1: overwrite, 0: accumulate into c (residual add, cuda/q_attn.cu:333)
    int unit_begin;  // filled by the launcher
    int strip_begin; // filled by the launcher
};

// ---- optional fusions around a launch (wgmma path) ----------------------------------------------------------------------
// RoPE applied in the epilogue of the matrices selected by `mask` (cuda/rope.cu:10-123 arithmetic; needs 128 % head_dim == 0
// so that a rotation partner lives in the same 128-column strip)
struct RopeFuse {
    const half* sin;
    const half* cos;
    const int32_t* past_lens;
    int past_len, q_len, head_dim, sincos_size, neox;
    unsigned mask;          // bit i: rotate mat[i]'s output
};
// A consumer of this launch's output: its activation buffer is filled directly from the epilogue, already permuted
// into the consumer's row order, in the wgmma core-matrix layout, times the consumer's RMSNorm weight -- the consumer
// launch then needs no prep kernel.  The RMSNorm's 1/rms is deferred: the producer leaves per-strip sums of squares
// in `sumsq`, the consumer multiplies its fp32 result by rsqrt(sum / K + eps).
struct ScatterTarget {
    half* xp;
    const uint16_t* invperm;    // consumer row of feature n (NULL: identity)
    const half* scale;          // RMSNorm weight (NULL: none)
};
struct GemvExtras {
    RopeFuse rope;                         // mask == 0: none
    ScatterTarget scat[GEMV_MAX_MATS];
    int num_scat;
    float* sumsq_out;                      // [strips][8] or NULL
    int prepared;                          // 1: mats[i].xp already hold the input (no prep launch)
    const float* sumsq_in;                 // with prepared: per-strip sums of squares of the input rows, or NULL (no norm)
    int sumsq_in_strips;
    float sumsq_eps;
};

struct GemvParams {
    GemvMat mat[GEMV_MAX_MATS];
    int num_mats;
    int M;                 // tokens this pass, 1..8 (8-wide tile) or 9..64 (wide tiles)
    int KS;                // slabs per strip (K/32), common to all matrices of the launch
    int total_units;       // sum over matrices of strips*KS
    const half* norm_w;    // fused RMSNorm weight (NULL: none): a = half(x * w * rsqrt(mean(x^2)+eps))
    float norm_eps;
    int epilogue;
    float* ws;             // split-K partial sums
    unsigned int* counters;
    int maxc;              // max contributors per strip (workspace stride)
    int act_stride;        // bytes between token rows of the staged activations in shared memory
    int act_rows;          // rows staged per segment (capacity)
    unsigned long long* dbg;   // optional phase timestamps (globaltimer) of CTA dbg_cta, NULL in production
    int dbg_cta;
    int tc_stage_bytes;    // wgmma kernel: bytes of one weight stage (largest group of one 32-column block)
    int tc_act_off;        // wgmma kernel: shared-memory offset of the staged activations
    int tc_act_bytes;      // wgmma kernel: bytes of the two activation rings
    int tc_stages;         // wgmma kernel: pipeline stages (groups in flight per warp), 2..4
    int row0;              // first token row of this pass (RoPE position bookkeeping)
    GemvExtras ex;
};

// Launch one or more passes (8 tokens each) of the GEMV over `nm` matrices that share K and the input layout.
// All matrices must live on `device`.  M may exceed 8 (extra passes re-read the weights, like the reference's
// grid.y = ceil(M/4) does, cuda/q_gemm.cu:97).  With `ex`, all M <= GEMV_MAX_CHAIN_ROWS rows run in one pass on the
// tc_tile(M)-wide kernel, reading and writing activation buffers in that tile's layout ([k / 8][tc_tile(M)][k % 8]).
int gemv_launch(int device, cudaStream_t stream, GemvMat* mats, int nm, int M, const half* norm_w, float norm_eps,
                int epilogue, const GemvExtras* ex = nullptr);
// Many-row path (gemm_big.cu): reconstruct a column window + cuBLAS fp16 GEMM with fp32 accumulation.  Un-chained launches
// of more than GEMM_BIG_MIN_ROWS rows take it (below, the packed-row kernels re-read the weights at most twice): row_path.
constexpr int GEMM_BIG_MIN_ROWS = 16;
bool gemm_big_available();
int gemm_big_launch(const QMatrix* q, const half* a, int lda, half* c, int ldc, int M, int clear, cudaStream_t stream);

// can `ex` be honoured for these matrices / this row count?  (LAYOUT_TC, one pass: up to 8 rows, or up to GEMV_MAX_CHAIN_ROWS
// when the launch is chained -- the un-chained block forms keep their 8-row passes above 8 rows)
bool gemv_supports_extras(const GemvMat* mats, int nm, int M, bool chained);
// can the wgmma kernel stage the matrix's quantisation groups (<= 4 KB per 32-column block)?
bool gemm_tc_supported(const QMatView& v);

// The kernel that runs one launch over the matrices qs[0..n) for `rows` rows (gemm_half_q_half and every block stage):
//   ROW_I8     one row, when the matrices can share one integer-GEMV launch (`i8_fusable`: the block handle's cached
//              gemv_i8_fusable, or LAYOUT_TC for a single matrix) and EXL2B_GEMV does not route rows to the wgmma kernel
//   ROW_DENSE  more than GEMM_BIG_MIN_ROWS rows, or groups the wgmma kernel cannot stage -- unless the launch is `chained`
//              (reads or writes another launch's activation buffer, which only the two row kernels do) or cuBLAS is missing
//   ROW_TC     otherwise: the wgmma kernel through gemv_launch
enum RowPath : int { ROW_I8, ROW_TC, ROW_DENSE };
RowPath row_path(int rows, const QMatrix* const* qs, int n, bool i8_fusable, bool chained);

}  // namespace exl2b
