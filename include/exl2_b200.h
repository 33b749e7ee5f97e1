/* exl2_b200.h -- C ABI of libexl2b200.so: the H100 (sm_90a) quantized-linear hot path of ExLlamaV2.
 *
 * Drop-in boundary (SURVEY.md 8b): the reference binds this path through the pybind11 module `exllamav2_ext`
 * (exllamav2/exllamav2_ext/ext_bindings.cpp:27-138).  Every entry point below names the reference binding it
 * replaces; exllamav2_b200/ext.py adapts torch.Tensor -> raw pointers and re-exports them under the reference's
 * own names, so exllamav2/{linear,attn,mlp,cache,rmsnorm}.py call it unchanged (see INTEGRATION.md).
 *
 * Conventions
 *   - plain C: raw device pointers, ints, an opaque cudaStream_t passed as void*; no torch types.
 *   - every function returns 0 on success, non-zero on error; exl2b_last_error() returns the message
 *     (the reference raises C++ exceptions via TORCH_CHECK, cpp/util.h:34-39; the shim raises RuntimeError).
 *   - "absent tensor" (the reference's meta-device none_tensor, ext.py:296) is a NULL pointer.
 *   - all launches go to the given stream; nothing on the forward path synchronises the device.
 *   - fp16 tensors are `uint16_t*` (IEEE binary16 bit patterns) to keep the header free of cuda_fp16.h.
 */
#ifndef EXL2_B200_H
#define EXL2_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* exl2b_stream_t;   /* cudaStream_t */
typedef void* exl2b_qmatrix_t;  /* opaque; the reference's QMatrix* handle (cuda/q_matrix.cuh:11-83) */
typedef void* exl2b_qattn_t;    /* reference QAttn*  (cuda/q_attn.cuh:38-171) */
typedef void* exl2b_qmlp_t;     /* reference QMLP*   (cuda/q_mlp.cuh) */

const char* exl2b_last_error(void);
int exl2b_version(void);
/* Number of kernels this library has launched since load (bench.py reports it as gpu_launches). */
uint64_t exl2b_launch_count(void);
/* 1 if single rows run on the integer GEMV (the default), 0 if on the wgmma kernel (EXL2B_GEMV=tc, read once at load).  A
 * chained single-row producer writes its consumer's input in the format of this path, so host code that picks the consumer
 * (the decode head) must follow it. */
int exl2b_row_gemv_i8(void);

/* ---- QMatrix ------------------------------------------------------------------------------------------------
 * replaces make_q_matrix (ext_qmatrix.cpp:21-111) / QMatrix::QMatrix (cuda/q_matrix.cu:49-196).
 * Exactly one of {q_scale,...} (EXL2) or {gptq_qzeros,...} (GPTQ) is non-NULL.
 * Like the reference (shuffle_kernel, q_matrix.cu:187-195) creation REWRITES q_weight in place into a private
 * layout (when width % 64 == 0; otherwise the handle owns a padded copy); q_scale/q_scale_max/qzeros/scales/
 * q_perm/bias stay owned by the caller and must outlive the handle (linear.py:145 keeps them alive).
 * q_scale_max must already carry the prescale/256 factor (ext.py:336).  q_groups may be a device or host pointer
 * (int16[2*groups]); gptq_g_idx is a HOST pointer (the reference passes w["g_idx"].cpu(), ext.py:385) or NULL;
 * for act-order GPTQ q_perm/q_invperm are caller-allocated device buffers that are FILLED here (ext.py:373-374,
 * q_matrix.cu:646-647).  temp_dq/max_dq_rows of the reference are not needed (no reconstruct+cuBLAS detour). */
typedef struct exl2b_qmatrix_desc {
    int device;
    int height;            /* K = in_features  */
    int width;             /* N = out_features */
    int groups;
    uint32_t* q_weight;    /* EXL2: int32[R, N];  GPTQ: qweight int32[K/8, N] */
    uint16_t* q_perm;      /* int16[K] or NULL (stored row k' <- input feature q_perm[k']) */
    uint16_t* q_invperm;   /* int16[K] or NULL */
    const uint32_t* q_scale;      /* EXL2 int32[G, N/8] */
    const uint16_t* q_scale_max;  /* EXL2 fp16[G], pre-multiplied by prescale/256 */
    const uint16_t* q_groups;     /* EXL2 int16[2G] (bits, first packed row) */
    int q_weight_rows;            /* EXL2: R (rows of q_weight) */
    const uint32_t* gptq_qzeros;  /* GPTQ int32[G, N/8] */
    const uint16_t* gptq_scales;  /* GPTQ fp16[G, N] */
    const int32_t* gptq_g_idx;    /* GPTQ int32[K] on the HOST, or NULL */
    const uint16_t* bias;         /* fp16[N] or NULL */
} exl2b_qmatrix_desc;

int exl2b_qmatrix_create(const exl2b_qmatrix_desc* desc, exl2b_stream_t stream, exl2b_qmatrix_t* out);
int exl2b_qmatrix_destroy(exl2b_qmatrix_t h);                     /* free_q_matrix, ext_qmatrix.cpp:187-194 */
int exl2b_qmatrix_info(exl2b_qmatrix_t h, int* height, int* width, int* groups, int* is_gptq, uint64_t* packed_bytes);
/* *supported = 1 if the wgmma kernel (2..16 rows, and every chained launch of 2..64 rows) can run this matrix: it stages one
 * quantisation group of a 32-column block at a time, at most 128 rows (4 KB at 8 bits).  Matrices with larger groups (EXL2 or
 * GPTQ g256+, ungrouped GPTQ) take the dense path at every row count above one instead, and cannot be chained there. */
int exl2b_qmatrix_tc_supported(exl2b_qmatrix_t h, int* supported);

/* reconstruct (ext_qmatrix.cpp:196-210, QMatrix::reconstruct q_matrix.cu:499-553):
 * out fp16[K, N] row-major in ORIGINAL row order, out[perm[k'], n] = half(q - zero) * half(scale), bit-exact. */
int exl2b_reconstruct(exl2b_qmatrix_t h, uint16_t* out, exl2b_stream_t stream);

/* gemm_half_q_half (ext_qmatrix.cpp:213-247 -> gemm_half_q_half_cuda, cuda/q_gemm.cu:201-313):
 * c[m, n] = (clear ? 0 : c[m, n]) + bias[n] + sum_k a[m, k] * W[k, n];  a fp16[M, K] (lda = row stride in
 * elements), c fp16[M, N] (ldc).  All M are served by the fused dequant kernels (no temp_dq, no cuBLAS);
 * force_cuda is accepted for signature parity and ignored. */
int exl2b_gemm_half_q_half(exl2b_qmatrix_t h, const uint16_t* a, int lda, uint16_t* c, int ldc, int m, int clear,
                           int force_cuda, exl2b_stream_t stream);

/* rms_norm (ext_norm.cpp:23-62) + gemm_half_q_half on ONE row as a single launch -- the final norm + lm_head of a decode
 * step (exllamav2/model.py:1036-1044 runs them as two kernels): c[n] = (clear ? 0 : c[n]) + bias[n] +
 * sum_k half(x[k] * w[k] * rsqrt(mean(x^2) + eps)) * W[k, n];  x fp16[K], c fp16[N]. */
int exl2b_gemm_half_q_half_norm(exl2b_qmatrix_t h, const uint16_t* x, const uint16_t* norm_w, float norm_eps, uint16_t* c,
                                int clear, exl2b_stream_t stream);

/* make_group_map (ext_qmatrix.cpp:341-361): host-only helper, out int16[2*K]; returns rows written / 2 in *k. */
int exl2b_make_group_map(const int16_t* q_groups, int num_groups, int num_qrows, int16_t* out, int out_capacity, int* k);

/* ---- RMSNorm / RoPE / activation ----------------------------------------------------------------------------
 * rms_norm / rms_norm_ (ext_norm.cpp:23-103 -> rms_norm_cuda, cuda/rms_norm.cu:177-229): y = x*w*rsqrt(mean(x^2)+eps),
 * fp16 in/out (y may alias x). */
int exl2b_rms_norm(const uint16_t* x, const uint16_t* w, uint16_t* y, float eps, int rows, int dim, exl2b_stream_t stream);

/* rope_ (ext_rope.cpp:20-62 -> rope_cuda, cuda/rope.cu:220-273): in-place rotary on x fp16[batch, rows_per_batch,
 * head_dim] where row = token*num_heads + head; position = past_len (+ past_lens[b], or past_lens[b] alone when
 * past_len == -1) + row / num_heads.  sin/cos fp16[max_pos, sincos_size]; neox != 0 -> half-split pairs. */
int exl2b_rope(uint16_t* x, const uint16_t* sin, const uint16_t* cos, int batch, int rows_per_batch, int head_dim,
               int num_heads, int past_len, const int32_t* past_lens, int neox, int sincos_size, exl2b_stream_t stream);

/* act_mul (cuda/q_mlp_activation.cuh:54-196): x = silu(x) * y (gelu when act_gelu), fp16, in place on x. */
int exl2b_act_mul(uint16_t* x, const uint16_t* y, int rows, int width, int act_gelu, exl2b_stream_t stream);

/* ---- Q4 / Q6 / Q8 K/V cache -------------------------------------------------------------------------------------
 * fp16_to_q_kv / q_to_fp16_kv (ext_cache.cpp:80-274 -> cuda/cache.cu:143-497, cuda/cache_q.cuh).  wbits = 4: keys and
 * values in 4 bits (uint8[..., dim/2] per row); 6: keys in 8 bits (uint8[..., dim]) and values in 4 bits; 8: both in 8 bits.
 * Scales are fp16[..., dim/32] in every format; any other wbits is an error.
 * Non-paged (page_size == 0): tensors are [batch, seq, heads*head_dim]; `dim` = heads*head_dim, `seq_stride` =
 * elements per batch row of the fp16 tensor; tokens [offset, offset+width) of every batch row are converted.
 * Paged (page_size > 0): block_table int32[batch, pages_per_seq], cache_seqlens int32[batch]; pack converts
 * tokens [seqlen, seqlen+q_len) (q_len passed in `width`), unpack converts [0, seqlen) of every sequence.
 * v_* may be NULL (single tensor). */
int exl2b_fp16_to_q_kv(const uint16_t* k_in, uint8_t* k_out, uint16_t* k_scales,
                       const uint16_t* v_in, uint8_t* v_out, uint16_t* v_scales,
                       int batch, int dim, int seq_stride, int offset, int width,
                       int page_size, const int32_t* cache_seqlens, const int32_t* block_table, int pages_per_seq,
                       int wbits, exl2b_stream_t stream);
int exl2b_q_to_fp16_kv(const uint8_t* k_in, const uint16_t* k_scales, uint16_t* k_out,
                       const uint8_t* v_in, const uint16_t* v_scales, uint16_t* v_out,
                       int batch, int dim, int seq_stride, int offset, int width,
                       int page_size, const int32_t* cache_seqlens, const int32_t* block_table, int pages_per_seq,
                       int wbits, exl2b_stream_t stream);

/* ---- fused attention / MLP blocks ---------------------------------------------------------------------------
 * make_q_attn / q_attn_forward_1 / q_attn_forward_2 (ext_qattn.cpp:24-191 -> cuda/q_attn.cu:153-345).
 * forward_1: RMSNorm(x) -> Q,K,V projections -> RoPE on Q and K; forward_2: x (+)= attn_out @ o_proj.
 * RMSNorm is folded into the projection kernel's prologue and Q/K/V run as ONE launch (SURVEY.md 7 step 3). */
typedef struct exl2b_qattn_desc {
    const uint16_t* layernorm;   /* fp16[hidden] RMSNorm weight or NULL; the single-row path reads a copy taken at create
                                    (here and in exl2b_qmlp_desc): recreate the handle after changing the weight */
    float norm_epsilon;
    exl2b_qmatrix_t q_proj, k_proj, v_proj, o_proj;
    int hidden_size, num_heads, num_kv_heads, head_dim;
    int has_residual;
    int rope_style;              /* 0 none, 1 gptj, 2 neox  (reference ROPE_STYLE_*, cuda/rope.cuh) */
    int sincos_size;
} exl2b_qattn_desc;
int exl2b_qattn_create(const exl2b_qattn_desc* desc, exl2b_qattn_t* out);
int exl2b_qattn_destroy(exl2b_qattn_t h);

/* make_q_mlp / q_mlp_forward_ (ext_qmlp.cpp:22-118 -> QMLP::forward_, cuda/q_mlp.cu:78-236):
 * x (+)= down( act(gate(norm(x))) * up(norm(x)) );  temp_a/temp_b fp16[rows, intermediate] scratch. */
typedef struct exl2b_qmlp_desc {
    const uint16_t* layernorm;
    float norm_epsilon;
    exl2b_qmatrix_t gate, up, down;
    int hidden_size, intermediate_size;
    int act_gelu;
    int has_residual;
} exl2b_qmlp_desc;
int exl2b_qmlp_create(const exl2b_qmlp_desc* desc, exl2b_qmlp_t* out);
int exl2b_qmlp_destroy(exl2b_qmlp_t h);
/* Column-sharded (tensor-parallel) use, exllamav2/tensor_p.py + ext_qattn.cpp:261-732 / ext_qmlp.cpp:326-473 in the
 * reference: a rank creates the attention block with ITS heads (num_heads / num_kv_heads = local counts) and o_proj = NULL,
 * the MLP block with ITS intermediate columns and down = NULL, runs part 1 / the gate|up half locally, all-gathers the
 * sharded activation, and applies its column shard of o_proj / down with exl2b_gemm_half_q_half(clear = 0) into its slice of
 * the residual stream (ldc = hidden size). */
int exl2b_qmlp_forward_gateup(exl2b_qmlp_t h, const uint16_t* x, int rows, uint16_t* temp_a, exl2b_stream_t stream);

/* ---- LoRA adapters on the blocks ------------------------------------------------------------------------------
 * q_attn_set_loras / q_mlp_set_loras (ext_qattn.cpp:194-240, ext_qmlp.cpp); a block forward's `ids` (below) are the active ones.
 * For every projection P with an adapter whose id is active: y_P += (in_P · A) · B, A fp16 [in_features, rank] and B fp16
 * [rank, out_features] (row-major, B already times the adapter's scaling, lora.py:168).  in_P is the RMSNorm'd block input for
 * q, k, v, gate and up (the delta lands before RoPE / act·mul), attn_output for o and act(gate)·up for down (the delta lands in
 * the residual stream after the projection has accumulated into it).  All active adapters of a projection are summed in fp32
 * and y is rounded to fp16 once.
 * A handle keeps the pointers, not copies: the tensors must outlive the set (the caller's adapter object owns them), and
 * in-place changes to their contents are seen by the next call, captured graphs included.
 * Projection index p: attention q 0, k 1, v 2, o 3; MLP gate 0, up 1, down 2. */
#define EXL2B_LORA_MAX_RANK 512      /* ranks (each rounded up to 8) of all adapters on one stage: q|k|v, o, gate|up or down */
#define EXL2B_LORA_MAX_ADAPTERS 8    /* adapters one handle holds */
typedef struct {
    uint64_t id;                     /* the caller's key (id(lora) in the reference) */
    const uint16_t* a[4];            /* per projection: A, or NULL for no adapter on it */
    const uint16_t* b[4];            /* B */
    int rank[4];
    int a_rows[4];                   /* in_features of A and out_features of B, checked against the projection's matrix */
    int b_cols[4];
} exl2b_lora_t;
/* Replace the handle's whole set (the reference clear()s, ext_qattn.cpp:208-211); *max_rank = the largest rank in it (the
 * reference's return value).  Rejects: A without B or B without A, shapes that do not match the matrix, a rank outside 1..512,
 * more than 8 adapters, an id given twice, and a set whose ranks would sum past EXL2B_LORA_MAX_RANK on any stage if all were
 * active at once. */
int exl2b_qattn_set_loras(exl2b_qattn_t h, const exl2b_lora_t* loras, int num, int* max_rank);
int exl2b_qmlp_set_loras(exl2b_qmlp_t h, const exl2b_lora_t* loras, int num, int* max_rank);
/* Host only: how one launch stacks the adapters.  ranks [num_adapters][num_projs] (0: none), all adapters active in order;
 * out per segment: its adapter, projection and first stacked column (each rank takes a multiple of 8 columns); *total = the
 * stacked width.  Fails, naming the bound, past EXL2B_LORA_MAX_RANK. */
int exl2b_lora_stack(const int* ranks, int num_adapters, int num_projs, int* seg_adapter, int* seg_proj, int* seg_off, int* num_segs,
                     int* total);

/* ---- block forwards -------------------------------------------------------------------------------------------
 * q_attn_forward_1 / q_attn_forward_2 / q_mlp_forward_ (ext_qattn.cpp:115-191, ext_qmlp.cpp:87-118 -> cuda/q_attn.cu:153-345,
 * cuda/q_mlp.cu:78-236, cuda/lora.cu): one entry point per stage -- q|k|v, o and the MLP -- with the reference's arguments and
 * three more.  input_prepared = 0, next = NULL and no ids make the reference's call.
 *
 * input_prepared, next -- chained launches (no reference counterpart: the reference runs norm / projection / rope / activation
 * as separate kernels).  A producer's epilogue can write its output straight into the activation buffer of the matrices that
 * consume it (`next`) -- permuted through their q_invperm, in the tensor-core operand layout, pre-multiplied by the RMSNorm
 * weight they apply -- together with per-strip sums of squares; the consumer launch (`input_prepared` = 1) then starts without
 * a prep kernel and applies 1/rms to its fp32 result, and does not read x (forward_1) or attn_out (forward_2) unless an adapter
 * is active (below).  Valid for rows <= 64 and the default (LAYOUT_TC) matrix layout with groups the wgmma kernel can stage
 * (exl2b_qmatrix_tc_supported); the calls fail otherwise.  Each launch runs its rows in one pass on the narrowest token tile
 * that holds them -- 8 (1..8 rows), 32 (9..32) or 64 (33..64) -- and a producer and its consumers must run the same row count:
 * 1..8 rows use the matrix's 8-row activation buffer, 9..64 rows a separate 64-row one.  `out_consumer` of
 * exl2b_paged_attn_decode_q is the same mechanism for the attention output (o_proj).
 *
 * ids, num_ids -- the call's active adapter ids (the reference's `loras`; NULL / 0 for none).  Ids registered nowhere on the
 * handle are skipped (cuda/lora.cu:20-21).  When no id has an adapter on a stage, that stage runs exactly as without adapters;
 * an adapted stage runs its base GEMMs with their raw outputs stored, then ONE LoRA launch (csrc/lora.cu) that adds every
 * adapter's delta and finishes the stage: RoPE of q and k, act(gate)·up, or nothing (o, down).
 *
 * Both -- a chained call with an active adapter runs each adapted stage as its chained base launch(es) followed by ONE LoRA
 * launch in the one-row form (csrc/lora.cu): it adds the deltas to the plain output row AND to the copy the base launch left in
 * the next consumer's stored-row order (the mirror), with the same bits, so the consumer reads the adapted row:
 *   q|k|v   q, k, v (no mirror: attention reads the plain rows; with sin / cos given the launch also applies RoPE);
 *   o       x, mirrored into next's first consumer (gate);
 *   gate|up the plain gate row (temp_a) and up row (temp_b), mirrored into down's input slots; no act·mul, down's prologue
 *           forms it;
 *   down    x, mirrored into next's first consumer (the next layer's q, or lm_head); its input act(gate)·up is formed from the
 *           two plain rows with the fp16 operations of down's own prologue.
 * The LoRA launches read x (q|k|v, gate|up) and attn_out (o) as plain rows in feature order, so neither may be NULL.  This holds
 * at ONE row on the integer GEMV only: above one row the chained launches fuse RoPE, act·mul and the RMSNorm sums of squares
 * into their epilogues, so no delta can be added after them -- such a call with an active adapter fails, saying so. */
typedef struct {
    exl2b_qmatrix_t consumers[3];   /* matrices whose INPUT is this launch's output (e.g. the next block's q, k, v) */
    int num_consumers;
    const uint16_t* norm_weight;    /* RMSNorm weight the consumers apply to that input, or NULL */
} exl2b_chain_t;
int exl2b_qattn_forward_1(exl2b_qattn_t h, const uint16_t* x, int batch, int q_len, int past_len, const int32_t* past_lens,
                          uint16_t* q, uint16_t* k, uint16_t* v, const uint16_t* sin, const uint16_t* cos,
                          int input_prepared, const uint64_t* ids, int num_ids, exl2b_stream_t stream);
int exl2b_qattn_forward_2(exl2b_qattn_t h, uint16_t* x, const uint16_t* attn_out, int batch, int q_len,
                          int input_prepared, const exl2b_chain_t* next, const uint64_t* ids, int num_ids, exl2b_stream_t stream);
int exl2b_qmlp_forward(exl2b_qmlp_t h, uint16_t* x, int rows, uint16_t* temp_a, uint16_t* temp_b,
                       int input_prepared, const exl2b_chain_t* next, const uint64_t* ids, int num_ids, exl2b_stream_t stream);
/* gemm_half_q_half on an input prepared by a chained producer (lm_head after the last MLP; has_norm: apply 1/rms) */
int exl2b_gemm_half_q_half_prepared(exl2b_qmatrix_t h, uint16_t* c, int ldc, int m, int clear, int has_norm, float norm_eps,
                                    exl2b_stream_t stream);

/* ---- host-buffer entry point (bench.py "e2e"): a fp16[M,K] and c fp16[M,N] are HOST pointers (pinned or
 * pageable); the call copies a to the device, runs gemm_half_q_half, copies c back and waits. */
int exl2b_gemm_half_q_half_host(exl2b_qmatrix_t h, const uint16_t* a_host, uint16_t* c_host, int m, exl2b_stream_t stream);

/* Tuning / diagnostics hook (no reference counterpart): CTAs per SM of the GEMV grid (<= 0 keeps the current value)
 * and an optional device buffer of 64 x 8 uint64 (one slot per launch, round robin): [0..5] globaltimer phase stamps of
 * CTA `cta`, [6] earliest CTA start (pre-fill with ~0), [7] latest CTA end (NULL disables). */
int exl2b_debug_set(int ctas_per_sm, unsigned long long* stamps, int cta);

/* Host-only diagnostics (no GPU needed): the 32-column-block -> CTA partition the batch-1 GEMV uses for blocks of the given
 * byte sizes; out[0..*used] are the block boundaries of the CTAs. */
int exl2b_debug_partition(const uint32_t* block_bytes, int num_blocks, int ctas, uint16_t* out, int* used);
/* diagnostics: per-CTA records (start, wait over, end, SM id) of the batch-1 GEMV launches, [64][160][4] uint64, or NULL */
int exl2b_debug_set_records(unsigned long long* records);
/* host-only: the per-warp stage lists of the batch-1 GEMV for one matrix structure (tests/test_i8_emulation.py) */
int exl2b_debug_plan(int N, int KS, int is_gptq, uint32_t blk_stream_bytes, const int* regions, int num_regions, int ctas, int warps,
                     int slot_bytes, uint32_t* desc, int cap_desc, uint32_t* first, int* ctas_used, int* n_desc, int* lcap,
                     uint32_t* red);
/* host-only: the whole batch-1 GEMV plan of a launch of nm fused matrices (arena, scale-slot size, shared memory, stage lists);
 * mats holds 5 + 5 * 6 ints per matrix: N, KS, is_gptq, blk_stream_bytes, num_regions, then (ks_begin, bits, spg_log2,
 * group_base, off_base) per region.  info: CTAs, descriptors, arena bytes, scale-slot bytes, shared-memory bytes, longest list. */
int exl2b_debug_i8_plan(const int* mats, int nm, int ctas, int warps, uint32_t* desc, int cap_desc, uint32_t* first, int cap_first,
                        int* info);
/* diagnostics: the device scratch a kernel family keeps for (device, stream) -- its address and size, or NULL / 0 before
 * the first launch that creates it.  Attention scratch is sized at its bound when created and never moves, so a graph
 * captured on the stream keeps valid pointers; the wgmma activation scratch (TC_XP) grows with the row count. */
enum {
    EXL2B_SCRATCH_ATTN_WS = 0,   /* split-KV partial results of the fused decode attention */
    EXL2B_SCRATCH_ATTN_CNT = 1,  /* its per-(sequence, head) arrival counters */
    EXL2B_SCRATCH_TC_WS = 2,     /* split-K workspace of the wgmma kernel */
    EXL2B_SCRATCH_TC_CNT = 3,    /* its arrival counters */
    EXL2B_SCRATCH_TC_XP = 4,     /* its activation-operand scratch */
    EXL2B_SCRATCH_TC_WS_WIDE = 5,   /* split-K workspace of the 32- and 64-row tiles (chained launches of 9..64 rows) */
    EXL2B_SCRATCH_TC_XP_WIDE = 6,   /* their activation-operand scratch; both created on the first such launch, never moved */
};
int exl2b_debug_scratch(int device, exl2b_stream_t stream, int kind, void** ptr, size_t* bytes);

/* Stand-in for flash_attn_with_kvcache (third-party in the reference, attn.py:602-613): appends the q_len new K/V rows
 * to the paged fp16 cache at [seqlen, seqlen+q_len) and attends causally.  q [batch,q_len,H,hd], k/v_new
 * [batch,q_len,KVH,hd], caches fp16 [pages,page_size,KVH,hd], out [batch,q_len,H,hd]; head_dim 64 or 128. */
int exl2b_paged_attn_decode(const uint16_t* q, const uint16_t* k_new, const uint16_t* v_new, uint16_t* k_cache,
                            uint16_t* v_cache, const int32_t* cache_seqlens, const int32_t* block_table, uint16_t* out,
                            int batch, int q_len, int num_heads, int num_kv_heads, int head_dim, int page_size,
                            int pages_per_seq, float softmax_scale, exl2b_stream_t stream);

/* Decode attention straight over the quantised cache (replaces the reference's per-layer sequence q_to_fp16_kv ->
 * flash_attn_with_kvcache -> fp16_to_q_kv, attn.py:560-613 + cache.py:472-556): quantises the q_len new K/V rows with
 * the fp16_to_q_kv arithmetic, appends them to the paged cache at [seqlen, seqlen+q_len) and attends causally over the
 * stored values.  `wbits` is the cache format, as for exl2b_fp16_to_q_kv: 4 (Q4), 6 (Q6 = 8-bit keys, 4-bit values) or 8 (Q8).
 * Shapes: q [batch,q_len,H,hd], k_new / v_new [batch,q_len,KVH,hd], out [batch,q_len,H,hd]; k_cache uint8
 * [pages,page_size,KVH,hd/2] for 4-bit keys and [...,hd] for 8-bit keys, v_cache likewise; k/v_scales fp16
 * [pages,page_size,KVH,hd/32]; 1 <= q_len <= 8; head_dim 64 or 128.
 * RoPE fused: when rope_style != 0 (1 gptj, 2 neox) and the tables are given, q and k_new are the UN-rotated projection
 * outputs and are rotated as they are read (rope_cuda arithmetic, cuda/rope.cu:52-67,111-122; position of row i =
 * cache_seqlens[b] + i), so q_attn_forward_1 can skip its rope launches (pass sin = cos = NULL there, rope_style = 0 for
 * none).  Needs sincos_size == head_dim.
 * `out_consumer` (or NULL): the matrix that takes the attention output (o_proj); the output is also left in its activation
 * buffer (chained launches, exl2b_chain_t) -- as a plain fp16 row in its stored-row order when there is a single row, where the
 * batch-1 GEMV reads it, and in the operand layout of the launch's token tile otherwise.  At most 64 rows (batch * q_len).
 * Cache length: with q_len 2..8 every CTA holds one fp32 score per position of its share of the cache's capacity
 * (pages_per_seq * page_size) in shared memory, so capacities above ~29 000 positions (hd 128) are refused ("context of N
 * tokens does not fit the score buffer").  A single-token step (q_len 1) whose scores do not fit walks each CTA's positions
 * in passes with an online softmax instead, and is refused only when the page table itself leaves no room for a pass of 512
 * positions (about 28 600 pages at Q4 hd 128), with an error naming the pages and the bytes (DESIGN.md §3.4). */
int exl2b_paged_attn_decode_q(const uint16_t* q, const uint16_t* k_new, const uint16_t* v_new, uint8_t* k_cache,
                              uint16_t* k_scales, uint8_t* v_cache, uint16_t* v_scales, const int32_t* cache_seqlens,
                              const int32_t* block_table, uint16_t* out, int batch, int q_len, int num_heads,
                              int num_kv_heads, int head_dim, int page_size, int pages_per_seq, float softmax_scale,
                              exl2b_qmatrix_t out_consumer, const uint16_t* rope_sin, const uint16_t* rope_cos,
                              int rope_style, int sincos_size, int wbits, exl2b_stream_t stream);
/* Prompt attention straight over the quantised cache, for any q_len >= 1 (replaces the reference's per-layer sequence for a
 * prompt chunk, q_to_fp16_kv -> flash_attn_with_kvcache -> fp16_to_q_kv, attn.py:560-621 + cache.py:472-556).  Same
 * semantics as exl2b_paged_attn_decode_q without fused RoPE or a chained output: query i of sequence b sees positions
 * [0, cache_seqlens[b] + i]; cached positions are the stored values, the q_len new positions are the UNQUANTISED fp16 k_new /
 * v_new rows (as flash-attn sees them in the reference, before the cache quantises them).  The new rows are quantised with the
 * fp16_to_q_kv arithmetic and appended at [seqlen, seqlen + q_len): only the new tokens' 64-value units are written, never
 * widened to 512-value blocks.  Tensor cores (mma.sync m16n8k16, fp16 operands, fp32 accumulation).
 * Shapes: q [batch,q_len,H,hd] (RoPE applied), k_new / v_new [batch,q_len,KVH,hd], out [batch,q_len,H,hd]; caches and scales as
 * for exl2b_paged_attn_decode_q; `wbits` 4 / 6 / 8; head_dim 64 or 128; H % KVH == 0; page_size a multiple of 64.
 * A sequence with cache_seqlens[b] + q_len > pages_per_seq * page_size gets no append and no output, and sets bit 0 of the
 * status below.  No host synchronisation and no allocation after the first call on a device: the launch can be captured. */
int exl2b_paged_attn_prefill_q(const uint16_t* q, const uint16_t* k_new, const uint16_t* v_new, uint8_t* k_cache,
                               uint16_t* k_scales, uint8_t* v_cache, uint16_t* v_scales, const int32_t* cache_seqlens,
                               const int32_t* block_table, uint16_t* out, int batch, int q_len, int num_heads,
                               int num_kv_heads, int head_dim, int page_size, int pages_per_seq, float softmax_scale,
                               int wbits, exl2b_stream_t stream);
/* Sticky status of the fused attention kernels on `device` (synchronises): bit 0 = a sequence would have run past its page
 * table (cache_seqlens[b] + q_len > pages_per_seq * page_size); that call appended nothing and wrote no output. */
int exl2b_paged_attn_status(int device, int* status);
int exl2b_paged_attn_clear_status(int device);

#ifdef __cplusplus
}
#endif
#endif /* EXL2_B200_H */
