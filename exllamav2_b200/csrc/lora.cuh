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
    int ld_act, gelu;
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
