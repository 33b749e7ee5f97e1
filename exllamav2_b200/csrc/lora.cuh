// LoRA adapters on the fused attention / MLP blocks (lora.cu): host interface shared with blocks.cu.
#pragma once
#include <vector>

#include "common.cuh"

namespace exl2b {

constexpr int LORA_MAX_RANK = EXL2B_LORA_MAX_RANK;          // stacked ranks of one launch (all its adapters and projections)
constexpr int LORA_MAX_ADAPTERS = EXL2B_LORA_MAX_ADAPTERS;  // adapters one handle holds
constexpr int LORA_MAX_SEGS = 3 * LORA_MAX_ADAPTERS;        // (adapter, projection) pairs of one launch
constexpr int LORA_MT = 8;                                  // rows per CTA (grid.y runs over row tiles)

// one adapter as a block handle holds it: per projection of the block (attention q, k, v, o; MLP gate, up, down) A fp16
// [K, rank] and B fp16 [rank, N] (B already times the adapter's scaling), or a = NULL
struct LoraProj {
    const half* a;
    const half* b;
    int rank;
};
struct LoraAdapter {
    uint64_t id;
    LoraProj p[4];
};

// one stacked (adapter, projection) pair of a launch: its ranks are columns [off, off + rank) of the launch's x·A
struct LoraSeg {
    const half* a;
    const half* b;
    int rank, off, proj;    // proj: index into the launch's outputs (LoraParams::y)
    int src;                // position of its adapter's id in the call's list
};

enum LoraEpilogue : int {
    LORA_ADD = 0,       // y[0] += delta                                            (o, down: the residual stream)
    LORA_QKV = 1,       // y[p] += delta for q, k, v; then RoPE on q and k          (rope_kernel arithmetic)
    LORA_ACT_MUL = 2,   // act_out = act(y[0] + delta_gate) * (y[1] + delta_up)   (act_mul_kernel arithmetic)
    LORA_ADD_PAIR = 3,  // y[0] += delta_gate, y[1] += delta_up, nothing more      (one-row form: down's prologue forms act·mul)
};

struct LoraParams {
    LoraSeg seg[LORA_MAX_SEGS];
    int nseg, R;                 // segments, stacked rank
    const half* x;               // input rows [rows][ldx] (ORIGINAL feature order)
    int ldx, K, rows;
    const half* norm_w;          // RMSNorm of the input rows (q|k|v, gate|up), or NULL
    float norm_eps;
    half* y[3];                  // the base GEMMs' outputs per projection of the launch, [rows][ldy]
    int n[3], ldy[3];
    int epi;
    int unit_pairs, units;       // column pairs per unit of work, units over the grid
    // LORA_QKV
    const half* sin;             // NULL: no rotation
    const half* cos;
    const int32_t* past_lens;
    int past_len, q_len, head_dim, sincos_size, neox, heads_q, heads_kv;
    // LORA_ACT_MUL
    half* act_out;
    int ld_act, gelu;            // gelu: also the activation of the x2 input below
    // input act(x) * x2 (x2 != NULL): the input row formed from the plain gate and up rows with I8_SILU_MUL / I8_GELU_MUL's fp16
    // operations (down's input in the chained single-row step, where the act·mul row never exists in memory)
    const half* x2;
    // one-row form (one_row = 1, rows = 1, no RoPE, epilogue ADD / QKV / ADD_PAIR): phase 3 spreads the stage's output columns
    // over all CTAs in groups of 8 (`groups` in all, set by lora_launch), each group's rank rows split between `tpg` threads
    // that read B 16 bytes at a time.  Every finished y[p][n] is also stored, same bits, at mirror[p][mirror_invperm[p][n]]
    // when mirror[p] is given: the copy a chained producer leaves in its consumer's stored-row order (I8Out::c_perm).
    int one_row, groups, tpg;
    half* mirror[3];
    const uint16_t* mirror_invperm[3];
};

// Stack the adapters of `ids` that have a projection in `projs` into p.seg (ids with none are skipped); -2 past the bounds.
int lora_stack(const std::vector<LoraAdapter>& ads, const uint64_t* ids, int num_ids, const int* projs, int nproj, LoraParams& p);
// Check and take a set of adapters for a block whose stages are `stages` (lists of projection indices, -1 ended); ks / ns:
// in / out features per projection.  Replaces `out`; *max_rank = largest rank of any projection.
int lora_take(const exl2b_lora_t* loras, int num, const int* ks, const int* ns, int nprojs, const int (*stages)[4], int nstages,
              std::vector<LoraAdapter>& out, int* max_rank);
// One cluster launch of the LoRA kernel over p (p.seg, p.x ... filled by the caller; grid and units here).
int lora_launch(int device, cudaStream_t stream, LoraParams& p);

}  // namespace exl2b
