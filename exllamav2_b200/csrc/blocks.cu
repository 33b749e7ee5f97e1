// Fused attention / MLP blocks behind make_q_attn / q_attn_forward_1 / q_attn_forward_2 (ext_qattn.cpp:24-191,
// cuda/q_attn.cu:153-345) and make_q_mlp / q_mlp_forward_ (ext_qmlp.cpp:22-118, cuda/q_mlp.cu:78-236).
//
// Launches per decoder layer for one decode row:  reference      here
//   attn part 1   norm, Q, K, V, rope              5              1  norm + Q|K|V in one GEMV launch (+ a rope launch for q
//                                                                    and one for k, unless the caller passes no sin/cos and
//                                                                    exl2b_paged_attn_decode_q rotates q / k as it reads them)
//   attn part 2   O (+residual via atomics)        1              1  residual add in the epilogue
//   mlp           norm, gate, up, act, down        5              2  norm + gate|up, then act*mul as down's prologue + residual
// The chained forms (input_prepared / next, exl2b_chain_t) have each launch write the next one's input in that matrix's
// stored-row order, and every launch carries the programmatic-dependent-launch attribute: the decode step captured in one CUDA
// graph (exllamav2_b200/model.py) is these 4 launches and attention per layer, streaming weights back to back.  A chained
// launch of 9..64 rows runs in one pass on the 32- or 64-row wgmma tile and feeds its consumers' 64-row activation buffers.
// Which kernel runs a stage (integer GEMV, wgmma, dense) is gemv.cu's row_path.
#include "gemv.cuh"
#include "gemv_i8.cuh"
#include "lora.cuh"

namespace exl2b {

int rope_launch(cudaStream_t stream, half* x, const half* sin, const half* cos, int batch, int rows_per_batch, int head_dim,
                int num_heads, int past_len, const int32_t* past_lens, int neox, int sincos_size);

struct QAttn {
    exl2b_qattn_desc d;
    int device;
    bool i8_qkv;          // q/k/v share K and the row permutation: one gemv_i8 launch for a single row
    half* norm_p;         // the layernorm in q/k/v's stored-row order, taken at creation (single-row launches), or NULL
    std::vector<LoraAdapter> loras;   // exl2b_qattn_set_loras: projections 0..3 = q, k, v, o
};
struct QMlp {
    exl2b_qmlp_desc d;
    int device;
    bool i8_gu;           // same for gate/up
    half* up_scratch;     // single-row up projection when the caller passes no temp_b (reference: temp_b of make_q_mlp)
    half* norm_p;         // the layernorm in gate/up's stored-row order, as QAttn::norm_p
    std::vector<LoraAdapter> loras;   // exl2b_qmlp_set_loras: projections 0..2 = gate, up, down
};

// the handle's copy of its layernorm in the stored-row order of the single-row GEMV's matrices (none without a permutation)
static int block_norm_copy(const QMatrix* q, const void* layernorm, bool i8, half** out) {
    *out = nullptr;
    if (!layernorm || !i8 || !q->v.perm) return 0;
    EXL2B_CUDA(cudaSetDevice(q->device));
    return permuted_norm_copy(q, (const half*)layernorm, out);
}

static GemvMat make_mat(const QMatrix* q, const half* x, int ldx, half* c, int ldc, int clear) {
    GemvMat m = {};
    m.w = q->v;
    m.x = x;
    m.ldx = ldx;
    m.c = c;
    m.ldc = ldc;
    m.clear = clear;
    return m;
}

// A chained launch of `rows` rows reads and writes the 8-row activation buffers (xp_buf / sumsq_buf) up to 8 rows, the 64-row
// ones (xp_wide / sumsq_wide) above
static half* chain_xp(const QMatrix* q, int rows) { return rows > GEMV_MTOK ? q->xp_wide : q->xp_buf; }
static float* chain_sumsq(const QMatrix* q, int rows) { return rows > GEMV_MTOK ? q->sumsq_wide : q->sumsq_buf; }

// epilogue of a producer launch -> the consumers' activation buffers (+ sums of squares when they apply an RMSNorm)
static int chain_out(GemvExtras& ex, const exl2b_chain_t* next, int rows) {
    if (!next || next->num_consumers <= 0) return 0;
    EXL2B_REQUIRE(next->num_consumers <= GEMV_MAX_MATS, "at most %d chained consumers", GEMV_MAX_MATS);
    for (int i = 0; i < next->num_consumers; ++i) {
        QMatrix* c = (QMatrix*)next->consumers[i];
        EXL2B_REQUIRE(c && c->v.layout == LAYOUT_TC, "chained consumer must be a LAYOUT_TC matrix");
        int rc = qmatrix_chain_buffers(c, rows > GEMV_MTOK);
        if (rc) return rc;
        ex.scat[i] = ScatterTarget{chain_xp(c, rows), c->invperm, (const half*)next->norm_weight};
    }
    ex.num_scat = next->num_consumers;
    if (next->norm_weight) ex.sumsq_out = chain_sumsq((QMatrix*)next->consumers[0], rows);
    return 0;
}
// consumer side: the matrices' inputs were written by a chained producer
static int chain_in(GemvExtras& ex, GemvMat* mats, const QMatrix* const* qs, int nm, bool has_norm, int rows) {
    ex.prepared = 1;
    for (int i = 0; i < nm; ++i) {
        EXL2B_REQUIRE(chain_xp(qs[i], rows), "input_prepared set, but no chained producer of %d rows has written this matrix's input",
                      rows);
        mats[i].xp = chain_xp(qs[i], rows);
    }
    if (has_norm) {
        ex.sumsq_in = chain_sumsq(qs[0], rows);
        ex.sumsq_in_strips = (qs[0]->v.K + 127) / 128;
    }
    return 0;
}

// i8 (single-row) form of a chain: the producer's finalisation scatters a second fp16 copy of its output into the first
// consumer's row buffer, in that matrix's stored-row order (all consumers of one chain share their permutation)
static int chain_out_i8(I8Out& o, const exl2b_chain_t* next, int slot = 0) {
    if (!next || next->num_consumers <= 0) return 0;
    QMatrix* c = (QMatrix*)next->consumers[0];
    EXL2B_REQUIRE(c && c->v.layout == LAYOUT_TC, "chained consumer must be a default-layout matrix");
    int rc = qmatrix_chain_buffers(c);
    if (rc) return rc;
    o.c_perm = c->xp_buf + (size_t)slot * c->v.K;
    o.out_invperm = c->invperm;
    return 0;
}

#define CHAIN_RULE "chained launches need LAYOUT_TC, at most %d rows and quantisation groups the wgmma kernel can stage " \
                   "(exl2b_qmatrix_tc_supported)"

// The integer GEMV's input row: x, or (chained) the row a producer launch left in q's stored-row order (I8Out::c_perm); the
// block's RMSNorm as the prologue when norm_w is given (norm_p: norm_w in that order, or NULL)
static int i8_input(I8Input& in, const uint16_t* x, bool chained, const QMatrix* q, const char* name, const uint16_t* norm_w,
                    float eps, const half* norm_p) {
    in = {(const half*)x, nullptr, (const half*)norm_w, eps, norm_w ? I8_RMSNORM : I8_PLAIN, 0, norm_p};
    if (chained) {
        EXL2B_REQUIRE(q->xp_buf, "input_prepared set, but no chained producer has written %s's input row", name);
        in.x = q->xp_buf;
        in.x_permuted = 1;
    }
    return 0;
}

// the handle's single-row buffer for the up projection when the caller passes no temp_b, allocated on first use
static int up_row(QMlp* m, half** out) {
    if (!m->up_scratch) EXL2B_CUDA(cudaMalloc(&m->up_scratch, (size_t)m->d.intermediate_size * sizeof(half)));
    *out = m->up_scratch;
    return 0;
}

// stand-alone RoPE of q and k (q_attn.cu:271-300)
static int rope_qk(const exl2b_qattn_desc& d, uint16_t* q, uint16_t* k, const uint16_t* sin, const uint16_t* cos, int batch,
                   int q_len, int past_len, const int32_t* past_lens, cudaStream_t stream) {
    const int neox = d.rope_style == 2;
    int rc = rope_launch(stream, (half*)q, (const half*)sin, (const half*)cos, batch, q_len * d.num_heads, d.head_dim, d.num_heads,
                         past_len, past_lens, neox, d.sincos_size);
    if (rc) return rc;
    return rope_launch(stream, (half*)k, (const half*)sin, (const half*)cos, batch, q_len * d.num_kv_heads, d.head_dim,
                       d.num_kv_heads, past_len, past_lens, neox, d.sincos_size);
}

// The dense path's GEMMs as the reference sequences them (q_attn.cu:153-300, q_mlp.cu:78-236): rms_norm into stream-ordered
// scratch, then out[i] = norm(x) @ qs[i] on the tensor cores (gemm_big.cu)
static int dense_gemms(const uint16_t* layernorm, float eps, const uint16_t* x, int rows, int hidden, const QMatrix* const* qs,
                       half* const* out, int n, cudaStream_t stream) {
    const half* xin = (const half*)x;
    half* xn = nullptr;
    int rc = 0;
    if (layernorm) {
        EXL2B_CUDA(cudaMallocAsync(&xn, (size_t)rows * hidden * sizeof(half), stream));
        rc = exl2b_rms_norm(x, layernorm, (uint16_t*)xn, eps, rows, hidden, (exl2b_stream_t)stream);
        xin = xn;
    }
    for (int i = 0; i < n && !rc; ++i) rc = gemm_big_launch(qs[i], xin, hidden, out[i], qs[i]->v.N, rows, 1, stream);
    if (xn) cudaFreeAsync(xn, stream);
    return rc;
}

// The q|k|v stage of batch * q_len rows.  raw = false: the finished q, k, v, RoPE applied -- fused into the wgmma epilogue where
// it fits, otherwise by rope_launch; on the integer GEMV a NULL sin skips it (exl2b_paged_attn_decode_q rotates q / k as it
// reads them).  raw = true: the projections alone, for the LoRA launch to finish.  chained: the input rows were left in the
// matrices' activation buffers by a producer launch (x is then unused).
static int qkv_stage(const QAttn* a, const uint16_t* x, int batch, int q_len, int past_len, const int32_t* past_lens, uint16_t* q,
                     uint16_t* k, uint16_t* v, const uint16_t* sin, const uint16_t* cos, bool chained, bool raw,
                     cudaStream_t stream) {
    const exl2b_qattn_desc& d = a->d;
    const int rows = batch * q_len;
    const QMatrix* qkv[3] = {(const QMatrix*)d.q_proj, (const QMatrix*)d.k_proj, (const QMatrix*)d.v_proj};
    half* out[3] = {(half*)q, (half*)k, (half*)v};
    const bool rope = d.rope_style != 0 && !raw;
    const RowPath path = row_path(rows, qkv, 3, a->i8_qkv, chained);
    int rc;
    if (path == ROW_I8) {
        // decode row: RMSNorm is the GEMV's prologue, Q|K|V are one launch (gemv_i8.cu)
        const I8Out o[3] = {{qkv[0], out[0], 1}, {qkv[1], out[1], 1}, {qkv[2], out[2], 1}};
        I8Input in;
        rc = i8_input(in, x, chained, qkv[0], "q_proj", d.layernorm, d.norm_epsilon, a->norm_p);
        if (!rc) rc = gemv_i8_launch(a->device, stream, o, 3, in);
        if (rc || !rope || !sin) return rc;
        return rope_qk(d, q, k, sin, cos, batch, q_len, past_len, past_lens, stream);
    }
    if (rope) EXL2B_REQUIRE(sin && cos, "rope needs sin/cos tables");
    if (path == ROW_DENSE) {
        rc = dense_gemms(d.layernorm, d.norm_epsilon, x, rows, d.hidden_size, qkv, out, 3, stream);
    } else {
        GemvMat mats[3];
        for (int i = 0; i < 3; ++i) mats[i] = make_mat(qkv[i], (const half*)x, d.hidden_size, out[i], qkv[i]->v.N, 1);
        const bool fuse = !raw && gemv_supports_extras(mats, 3, rows, chained) &&
                          (!rope || (d.head_dim <= 128 && 128 % d.head_dim == 0 && d.sincos_size <= d.head_dim));
        EXL2B_REQUIRE(!chained || fuse, CHAIN_RULE, GEMV_MAX_CHAIN_ROWS);
        if (fuse) {
            GemvExtras ex = {};
            if (rope) ex.rope = RopeFuse{(const half*)sin, (const half*)cos, past_lens, past_len, q_len, d.head_dim, d.sincos_size, d.rope_style == 2, 3u};
            if (chained) {
                rc = chain_in(ex, mats, qkv, 3, d.layernorm != nullptr, rows);
                if (rc) return rc;
            }
            return gemv_launch(a->device, stream, mats, 3, rows, (const half*)d.layernorm, d.norm_epsilon, EPI_STORE, &ex);
        }
        rc = gemv_launch(a->device, stream, mats, 3, rows, (const half*)d.layernorm, d.norm_epsilon, EPI_STORE);
    }
    if (rc || !rope) return rc;
    return rope_qk(d, q, k, sin, cos, batch, q_len, past_len, past_lens, stream);
}

// The gate|up stage of `rows` rows on `path` (never chained).  act = true: temp_a = act(gate) * up, with up through `up` or
// (NULL) through scratch.  act = false: raw gate -> temp_a, raw up -> `up` (given), for the LoRA launch to finish.
static int gate_up_stage(QMlp* m, RowPath path, const uint16_t* x, int rows, uint16_t* temp_a, half* up, bool act,
                         cudaStream_t stream) {
    const exl2b_qmlp_desc& d = m->d;
    const QMatrix* gu[2] = {(const QMatrix*)d.gate, (const QMatrix*)d.up};
    int rc = 0;
    if (path == ROW_I8) {
        // decode row: gate|up as one integer-GEMV launch with RMSNorm as its prologue
        if (!up) {
            rc = up_row(m, &up);
            if (rc) return rc;
        }
        const I8Out o[2] = {{gu[0], (half*)temp_a, 1}, {gu[1], up, 1}};
        I8Input in;
        rc = i8_input(in, x, false, gu[0], "gate_proj", d.layernorm, d.norm_epsilon, m->norm_p);
        if (!rc) rc = gemv_i8_launch(m->device, stream, o, 2, in);
        if (rc || !act) return rc;
        return exl2b_act_mul(temp_a, (const uint16_t*)up, 1, d.intermediate_size, d.act_gelu, (exl2b_stream_t)stream);
    }
    if (path == ROW_DENSE) {
        half* tb = up;
        if (!tb) EXL2B_CUDA(cudaMallocAsync(&tb, (size_t)rows * d.intermediate_size * sizeof(half), stream));
        half* out[2] = {(half*)temp_a, tb};
        rc = dense_gemms(d.layernorm, d.norm_epsilon, x, rows, d.hidden_size, gu, out, 2, stream);
        if (!rc && act) rc = exl2b_act_mul(temp_a, (const uint16_t*)tb, rows, d.intermediate_size, d.act_gelu, (exl2b_stream_t)stream);
        if (!up) cudaFreeAsync(tb, stream);
        return rc;
    }
    // the wgmma kernel, act(gate) * up formed in its epilogue
    GemvMat mats[2] = {
        make_mat(gu[0], (const half*)x, d.hidden_size, (half*)temp_a, d.intermediate_size, 1),
        make_mat(gu[1], (const half*)x, d.hidden_size, act ? (half*)temp_a : up, d.intermediate_size, 1),
    };
    return gemv_launch(m->device, stream, mats, 2, rows, (const half*)d.layernorm, d.norm_epsilon,
                       !act ? EPI_STORE : d.act_gelu ? EPI_GELU_MUL : EPI_SILU_MUL);
}


// A launch is chained when its input was left in its matrices' activation buffers by a producer launch (input_prepared) or
// it leaves its output in the buffers of next's consumers
static bool is_chained(int input_prepared, const exl2b_chain_t* next) {
    return input_prepared || (next && next->num_consumers > 0);
}

// The o stage of `rows` rows: x (+)= attn_out @ o_proj.  Chained, the input row is read from o_proj's activation buffer
// (input_prepared: attn_out is unused) and the output also goes to next's consumers.
static int o_stage(const QAttn* a, uint16_t* x, const uint16_t* attn_out, int rows, int input_prepared, const exl2b_chain_t* next,
                   cudaStream_t stream) {
    const QMatrix* mo = (const QMatrix*)a->d.o_proj;
    const int clear = a->d.has_residual ? 0 : 1;
    const bool chained = is_chained(input_prepared, next);
    const RowPath path = row_path(rows, &mo, 1, mo->v.layout == LAYOUT_TC, chained);
    if (path == ROW_I8) {
        I8Out o = {mo, (half*)x, clear};
        I8Input in;
        int rc = i8_input(in, attn_out, input_prepared, mo, "o_proj", nullptr, 0.f, nullptr);
        if (!rc) rc = chain_out_i8(o, next);
        if (rc) return rc;
        return gemv_i8_launch(a->device, stream, &o, 1, in);
    }
    if (path == ROW_DENSE) return gemm_big_launch(mo, (const half*)attn_out, mo->v.K, (half*)x, mo->v.N, rows, clear, stream);
    GemvMat m = make_mat(mo, (const half*)attn_out, mo->v.K, (half*)x, mo->v.N, clear);
    if (!chained) return gemv_launch(a->device, stream, &m, 1, rows, nullptr, 0.f, EPI_STORE);
    EXL2B_REQUIRE(gemv_supports_extras(&m, 1, rows, true), CHAIN_RULE, GEMV_MAX_CHAIN_ROWS);
    GemvExtras ex = {};
    int rc = chain_out(ex, next, rows);
    if (rc) return rc;
    if (input_prepared) {
        rc = chain_in(ex, &m, &mo, 1, false, rows);
        if (rc) return rc;
    }
    return gemv_launch(a->device, stream, &m, 1, rows, nullptr, 0.f, EPI_STORE, &ex);
}

// ---- LoRA adapters (lora.cu) ------------------------------------------------------------------------------------------------------
// An adapted stage runs its base GEMMs on the kernel row_path picks, with the raw outputs stored, then one LoRA launch that adds
// the deltas and finishes the stage.  A stage with no active adapter runs exactly as without adapters.  The launch covers all
// rows of an un-chained call, or takes the one-row form in a chained single-row call (the helpers below: `mirror` given).

static const int ATTN_STAGES[2][4] = {{0, 1, 2, -1}, {3, -1, -1, -1}};
static const int MLP_STAGES[2][4] = {{0, 1, -1, -1}, {2, -1, -1, -1}};

// Adapters on a chained call: the LoRA launch adds its deltas after the producer, which needs the single-row integer GEMV
static int lora_chain_rule(int rows, RowPath path) {
    EXL2B_REQUIRE(rows == 1,
                  "LoRA adapters on a chained call of %d rows: above one row the chained launches fuse RoPE, act(gate)*up and the "
                  "RMSNorm sums of squares into their epilogues, so no delta can be added after them (use the un-chained forms)",
                  rows);
    EXL2B_REQUIRE(path == ROW_I8, "LoRA adapters on a chained call need the single-row integer GEMV (not EXL2B_GEMV=tc)");
    return 0;
}

// The one-row form: output p's delta also goes, same bits, to the copy its base launch left in the next consumer's stored-row
// order (mirror[p].c_perm, chain_out_i8; NULL: no copy)
static void lora_one_row(LoraParams& lp, const I8Out* mirror, int np) {
    lp.one_row = 1;
    for (int p = 0; p < np; ++p) {
        lp.mirror[p] = mirror[p].c_perm;
        lp.mirror_invperm[p] = mirror[p].out_invperm;
    }
}

// The adapted q|k|v stage (lp: its stacked adapters): the raw projections, then the LoRA launch that adds the deltas and applies
// RoPE.  chained: the base launch reads the row a producer left in q's activation buffer (one row); x, the same row in feature
// order, is the LoRA launch's input.  Without RoPE there the launch takes the one-row form and attention rotates q and k.
static int qkv_lora(QAttn* a, LoraParams& lp, const uint16_t* x, int batch, int q_len, int past_len, const int32_t* past_lens,
                    uint16_t* q, uint16_t* k, uint16_t* v, const uint16_t* sin, const uint16_t* cos, bool chained,
                    cudaStream_t stream) {
    const exl2b_qattn_desc& d = a->d;
    const int rows = batch * q_len;
    const bool rope = d.rope_style != 0 && sin;
    if (d.rope_style != 0 && rows > 1) EXL2B_REQUIRE(sin && cos, "rope needs sin/cos tables");
    int rc = qkv_stage(a, x, batch, q_len, past_len, past_lens, q, k, v, sin, cos, chained, true, stream);
    if (rc) return rc;
    lp.one_row = chained && !rope;
    lp.x = (const half*)x;
    lp.ldx = lp.K = d.hidden_size;
    lp.rows = rows;
    lp.norm_w = (const half*)d.layernorm;
    lp.norm_eps = d.norm_epsilon;
    const QMatrix* qkv[3] = {(const QMatrix*)d.q_proj, (const QMatrix*)d.k_proj, (const QMatrix*)d.v_proj};
    half* ys[3] = {(half*)q, (half*)k, (half*)v};
    for (int p = 0; p < 3; ++p) {
        lp.y[p] = ys[p];
        lp.n[p] = lp.ldy[p] = qkv[p]->v.N;
    }
    lp.epi = LORA_QKV;
    lp.head_dim = d.head_dim;
    lp.heads_q = d.num_heads;
    lp.heads_kv = d.num_kv_heads;
    if (rope) {
        EXL2B_REQUIRE(d.head_dim % 2 == 0 && d.sincos_size % 4 == 0 && d.sincos_size <= d.head_dim, "rope: bad head_dim/sincos_size");
        lp.sin = (const half*)sin;
        lp.cos = (const half*)cos;
        lp.past_lens = past_lens;
        lp.past_len = past_len;
        lp.q_len = q_len;
        lp.sincos_size = d.sincos_size;
        lp.neox = d.rope_style == 2;
    }
    return lora_launch(a->device, stream, lp);
}

// o's LoRA launch, after its base launch: x += attn_out · A · B
static int o_lora(const QAttn* a, LoraParams& lp, uint16_t* x, const uint16_t* attn_out, int rows, const I8Out* mirror,
                  cudaStream_t stream) {
    const QMatrix* mo = (const QMatrix*)a->d.o_proj;
    lp.x = (const half*)attn_out;
    lp.ldx = lp.K = mo->v.K;
    lp.rows = rows;
    lp.y[0] = (half*)x;
    lp.n[0] = lp.ldy[0] = mo->v.N;
    lp.epi = LORA_ADD;
    if (mirror) lora_one_row(lp, mirror, 1);
    return lora_launch(a->device, stream, lp);
}

// gate|up's LoRA launch, after the raw gate (temp_a) and up rows: temp_a = act(gate + delta) * (up + delta).  The one-row form
// adds the deltas to both rows and their copies in down's input slots, and stops there: down's prologue forms act·mul.
static int gate_up_lora(const QMlp* m, LoraParams& lp, const uint16_t* x, int rows, uint16_t* temp_a, half* up, const I8Out* mirror,
                        cudaStream_t stream) {
    const exl2b_qmlp_desc& d = m->d;
    lp.x = (const half*)x;
    lp.ldx = lp.K = d.hidden_size;
    lp.rows = rows;
    lp.norm_w = (const half*)d.layernorm;
    lp.norm_eps = d.norm_epsilon;
    lp.y[0] = (half*)temp_a;
    lp.y[1] = up;
    lp.n[0] = lp.n[1] = lp.ldy[0] = lp.ldy[1] = d.intermediate_size;
    if (mirror) {
        lp.epi = LORA_ADD_PAIR;
        lora_one_row(lp, mirror, 2);
    } else {
        lp.epi = LORA_ACT_MUL;
        lp.act_out = (half*)temp_a;
        lp.ld_act = d.intermediate_size;
        lp.gelu = d.act_gelu;
    }
    return lora_launch(m->device, stream, lp);
}

// down's LoRA launch, after its base launch: x += temp_a · A · B, temp_a = act(gate)·up.  In the one-row form that row never
// exists in memory: the launch forms it from the plain gate row (temp_a) and up row (x2) with the fp16 operations of down's
// prologue.
static int down_lora(const QMlp* m, LoraParams& lp, uint16_t* x, const uint16_t* temp_a, const half* x2, int rows,
                     const I8Out* mirror, cudaStream_t stream) {
    const exl2b_qmlp_desc& d = m->d;
    lp.x = (const half*)temp_a;
    lp.ldx = lp.K = d.intermediate_size;
    lp.rows = rows;
    lp.y[0] = (half*)x;
    lp.n[0] = lp.ldy[0] = d.hidden_size;
    lp.epi = LORA_ADD;
    if (mirror) {
        lp.x2 = x2;
        lp.gelu = d.act_gelu;
        lora_one_row(lp, mirror, 1);
    }
    return lora_launch(m->device, stream, lp);
}

// The single-row MLP on the integer GEMV: gate|up in one launch with RMSNorm as its prologue; act(gate) * up is the PROLOGUE of
// the down launch, which reads both rows in its own stored-row order (scattered there by the gate|up launch's finalisation).
// gu / dn (or NULL): the stages' LoRA launches, each after its base launch, in the one-row form: gate|up's adds its deltas to
// both rows and to down's copies of them, down's forms act(gate)·up from the plain rows and adds to x and to next's copy.
static int mlp_row(QMlp* m, uint16_t* x, uint16_t* temp_a, uint16_t* temp_b, int input_prepared, const exl2b_chain_t* next,
                   LoraParams* gu, LoraParams* dn, cudaStream_t stream) {
    const exl2b_qmlp_desc& d = m->d;
    const QMatrix *g = (const QMatrix*)d.gate, *u = (const QMatrix*)d.up, *dm = (const QMatrix*)d.down;
    half* tb = (half*)temp_b;
    int rc = tb ? 0 : up_row(m, &tb);
    if (!rc) rc = qmatrix_chain_buffers(const_cast<QMatrix*>(dm));
    if (rc) return rc;
    I8Out o[2] = {{g, (half*)temp_a, 1}, {u, tb, 1}};
    o[0].c_perm = dm->xp_buf;
    o[1].c_perm = dm->xp_buf + dm->v.K;
    o[0].out_invperm = o[1].out_invperm = dm->invperm;
    I8Input in1;
    rc = i8_input(in1, x, input_prepared, g, "gate_proj", d.layernorm, d.norm_epsilon, m->norm_p);
    if (!rc) rc = gemv_i8_launch(m->device, stream, o, 2, in1);
    if (!rc && gu && gu->nseg) rc = gate_up_lora(m, *gu, x, 1, temp_a, tb, o, stream);
    if (rc) return rc;
    I8Out od = {dm, (half*)x, d.has_residual ? 0 : 1};
    rc = chain_out_i8(od, next);
    if (rc) return rc;
    const I8Input in2 = {dm->xp_buf, dm->xp_buf + dm->v.K, nullptr, 0.f, d.act_gelu ? I8_GELU_MUL : I8_SILU_MUL, 1};
    rc = gemv_i8_launch(m->device, stream, &od, 1, in2);
    if (rc || !dn || !dn->nseg) return rc;
    return down_lora(m, *dn, x, temp_a, tb, 1, &od, stream);
}

// The MLP without adapters on the path row_path picks for its three matrices: mlp_row for one row, otherwise gate|up then down
// (+residual), the two fused through down's activation buffer when the wgmma kernel runs both
static int mlp_stages(QMlp* m, uint16_t* x, int rows, uint16_t* temp_a, uint16_t* temp_b, int input_prepared,
                      const exl2b_chain_t* next, cudaStream_t stream) {
    const exl2b_qmlp_desc& d = m->d;
    const QMatrix *g = (const QMatrix*)d.gate, *u = (const QMatrix*)d.up, *dn = (const QMatrix*)d.down;
    const QMatrix* gud[3] = {g, u, dn};
    const bool chained = is_chained(input_prepared, next);
    const RowPath path = row_path(rows, gud, 3, m->i8_gu && dn->v.layout == LAYOUT_TC, chained);
    if (path == ROW_I8) return mlp_row(m, x, temp_a, temp_b, input_prepared, next, nullptr, nullptr, stream);
    GemvMat gu[2] = {
        make_mat(g, (const half*)x, d.hidden_size, (half*)temp_a, d.intermediate_size, 1),
        make_mat(u, (const half*)x, d.hidden_size, (half*)temp_a, d.intermediate_size, 1),
    };
    GemvMat down = make_mat(dn, (const half*)temp_a, d.intermediate_size, (half*)x, d.hidden_size, d.has_residual ? 0 : 1);
    const bool fuse = path == ROW_TC && gemv_supports_extras(gu, 2, rows, chained) && gemv_supports_extras(&down, 1, rows, chained);
    EXL2B_REQUIRE(fuse || !chained, CHAIN_RULE, GEMV_MAX_CHAIN_ROWS);
    if (!fuse) {
        // act(gate) * up into temp_a, then down (+residual): on the dense path as in q_mlp.cu:78-236, or on the wgmma kernel
        int rc = gate_up_stage(m, path, x, rows, temp_a, (half*)temp_b, true, stream);
        if (rc) return rc;
        if (path == ROW_DENSE)
            return gemm_big_launch(dn, (const half*)temp_a, d.intermediate_size, (half*)x, d.hidden_size, rows, down.clear, stream);
        return gemv_launch(m->device, stream, &down, 1, rows, nullptr, 0.f, EPI_STORE);
    }
    // gate|up writes silu(gate)*up straight into down's activation buffer (permuted, core-matrix layout): no prep launch between
    GemvExtras e1 = {};
    exl2b_chain_t to_down = {};
    to_down.consumers[0] = (exl2b_qmatrix_t)dn;
    to_down.num_consumers = 1;
    int rc = chain_out(e1, &to_down, rows);
    if (rc) return rc;
    if (input_prepared) {
        const QMatrix* qs[2] = {g, u};
        rc = chain_in(e1, gu, qs, 2, d.layernorm != nullptr, rows);
        if (rc) return rc;
    }
    rc = gemv_launch(m->device, stream, gu, 2, rows, (const half*)d.layernorm, d.norm_epsilon,
                     d.act_gelu ? EPI_GELU_MUL : EPI_SILU_MUL, &e1);
    if (rc) return rc;
    GemvExtras e2 = {};
    rc = chain_out(e2, next, rows);
    if (rc) return rc;
    rc = chain_in(e2, &down, &dn, 1, false, rows);
    if (rc) return rc;
    return gemv_launch(m->device, stream, &down, 1, rows, nullptr, 0.f, EPI_STORE, &e2);
}

// The un-chained MLP with adapters (gu / dn: the stacked adapters of gate|up and of down; one of them may have none).  An adapted
// gate|up stores raw gate -> temp_a and raw up -> temp_b, and its LoRA launch writes act(gate + delta) * (up + delta) over temp_a;
// otherwise gate|up forms act(gate) * up itself.  Down is gemm_half_q_half on temp_a, then its LoRA launch when adapted.
static int mlp_lora(QMlp* m, uint16_t* x, int rows, uint16_t* temp_a, uint16_t* temp_b, LoraParams& gu, LoraParams& dn,
                    cudaStream_t stream) {
    const exl2b_qmlp_desc& d = m->d;
    const QMatrix* gu2[2] = {(const QMatrix*)d.gate, (const QMatrix*)d.up};
    const RowPath path = row_path(rows, gu2, 2, m->i8_gu, false);
    int rc;
    if (gu.nseg) {
        half* tb = (half*)temp_b;
        bool own_tb = false;
        if (!tb && rows == 1) {
            rc = up_row(m, &tb);
            if (rc) return rc;
        } else if (!tb) {
            EXL2B_CUDA(cudaMallocAsync(&tb, (size_t)rows * d.intermediate_size * sizeof(half), stream));
            own_tb = true;
        }
        rc = gate_up_stage(m, path, x, rows, temp_a, tb, false, stream);
        if (!rc) rc = gate_up_lora(m, gu, x, rows, temp_a, tb, nullptr, stream);
        if (own_tb) cudaFreeAsync(tb, stream);
    } else {
        rc = gate_up_stage(m, path, x, rows, temp_a, nullptr, true, stream);          // temp_a = act(gate) * up
    }
    if (rc) return rc;
    rc = exl2b_gemm_half_q_half(d.down, temp_a, d.intermediate_size, x, d.hidden_size, rows, d.has_residual ? 0 : 1, 0,
                                (exl2b_stream_t)stream);
    if (rc || dn.nseg == 0) return rc;
    return down_lora(m, dn, x, temp_a, nullptr, rows, nullptr, stream);
}

}  // namespace exl2b

using namespace exl2b;

extern "C" int exl2b_qattn_create(const exl2b_qattn_desc* d, exl2b_qattn_t* out) {
    EXL2B_REQUIRE(d && out, "null argument");
    // o_proj may be absent: a tensor-parallel rank runs part 1 on its heads and applies its column shard of o_proj itself
    // (exllamav2_b200/tensor_p.py), part 2 then is not available on this handle
    EXL2B_REQUIRE(d->q_proj && d->k_proj && d->v_proj, "q/k/v handles are required");
    const QMatrix *q = (const QMatrix*)d->q_proj, *k = (const QMatrix*)d->k_proj, *v = (const QMatrix*)d->v_proj,
                  *o = d->o_proj ? (const QMatrix*)d->o_proj : q;
    EXL2B_REQUIRE(q->v.K == d->hidden_size && k->v.K == d->hidden_size && v->v.K == d->hidden_size, "q/k/v_proj is wrong shape");
    EXL2B_REQUIRE(!d->o_proj || o->v.N == d->hidden_size, "o_proj is wrong shape");          // ext_qattn.cpp:67
    EXL2B_REQUIRE(q->v.N == d->num_heads * d->head_dim && k->v.N == d->num_kv_heads * d->head_dim && v->v.N == k->v.N,
                  "projection widths do not match the head layout");
    EXL2B_REQUIRE(q->device == k->device && q->device == v->device && q->device == o->device, "handles on different devices");
    const QMatrix* qkv[3] = {q, k, v};
    const bool i8 = gemv_i8_fusable(qkv, 3);
    half* norm_p = nullptr;
    int rc = block_norm_copy(q, d->layernorm, i8, &norm_p);
    if (rc) return rc;
    QAttn* a = new QAttn{*d, q->device, i8, norm_p};
    *out = (exl2b_qattn_t)a;
    return 0;
}

extern "C" int exl2b_qattn_destroy(exl2b_qattn_t h) {
    QAttn* a = (QAttn*)h;
    if (a && a->norm_p) {
        cudaSetDevice(a->device);
        cudaFree(a->norm_p);
    }
    delete a;
    return 0;
}

extern "C" int exl2b_qattn_forward_1(exl2b_qattn_t h, const uint16_t* x, int batch, int q_len, int past_len,
                                     const int32_t* past_lens, uint16_t* q, uint16_t* k, uint16_t* v, const uint16_t* sin,
                                     const uint16_t* cos, int input_prepared, const uint64_t* ids, int num_ids,
                                     exl2b_stream_t stream_) {
    QAttn* a = (QAttn*)h;
    EXL2B_REQUIRE(a && q && k && v && (x || input_prepared) && (ids || num_ids == 0), "null argument");
    LoraParams lp = {};
    int rc = lora_stack(a->loras, ids, num_ids, ATTN_STAGES[0], 3, lp);
    if (rc) return rc;
    EXL2B_CUDA(cudaSetDevice(a->device));
    cudaStream_t stream = (cudaStream_t)stream_;
    if (lp.nseg == 0)
        return qkv_stage(a, x, batch, q_len, past_len, past_lens, q, k, v, sin, cos, input_prepared != 0, false, stream);
    if (!input_prepared) return qkv_lora(a, lp, x, batch, q_len, past_len, past_lens, q, k, v, sin, cos, false, stream);
    const QMatrix* qkv[3] = {(const QMatrix*)a->d.q_proj, (const QMatrix*)a->d.k_proj, (const QMatrix*)a->d.v_proj};
    rc = lora_chain_rule(batch * q_len, row_path(batch * q_len, qkv, 3, a->i8_qkv, true));
    if (rc) return rc;
    EXL2B_REQUIRE(x, "LoRA adapters on a chained q|k|v: the LoRA launch reads the block input x, which the producer also leaves there");
    return qkv_lora(a, lp, x, batch, q_len, past_len, past_lens, q, k, v, sin, cos, true, stream);
}

extern "C" int exl2b_qattn_forward_2(exl2b_qattn_t h, uint16_t* x, const uint16_t* attn_out, int batch, int q_len,
                                     int input_prepared, const exl2b_chain_t* next, const uint64_t* ids, int num_ids,
                                     exl2b_stream_t stream_) {
    QAttn* a = (QAttn*)h;
    EXL2B_REQUIRE(a && x && (attn_out || input_prepared) && (ids || num_ids == 0), "null argument");
    LoraParams lp = {};
    int rc = lora_stack(a->loras, ids, num_ids, ATTN_STAGES[1], 1, lp);
    if (rc) return rc;
    EXL2B_REQUIRE(a->d.o_proj, "this attention handle was created without o_proj");
    EXL2B_CUDA(cudaSetDevice(a->device));
    cudaStream_t stream = (cudaStream_t)stream_;
    const int rows = batch * q_len;
    if (lp.nseg == 0) return o_stage(a, x, attn_out, rows, input_prepared, next, stream);
    if (!is_chained(input_prepared, next)) {
        rc = o_stage(a, x, attn_out, rows, 0, nullptr, stream);
        return rc ? rc : o_lora(a, lp, x, attn_out, rows, nullptr, stream);
    }
    const QMatrix* mo = (const QMatrix*)a->d.o_proj;
    rc = lora_chain_rule(rows, row_path(rows, &mo, 1, mo->v.layout == LAYOUT_TC, true));
    if (rc) return rc;
    EXL2B_REQUIRE(attn_out, "LoRA adapters on a chained o_proj: the LoRA launch reads attn_out, which attention also writes");
    I8Out mirror = {};
    rc = o_stage(a, x, attn_out, rows, input_prepared, next, stream);
    if (!rc) rc = chain_out_i8(mirror, next);
    return rc ? rc : o_lora(a, lp, x, attn_out, rows, &mirror, stream);
}

extern "C" int exl2b_qmlp_create(const exl2b_qmlp_desc* d, exl2b_qmlp_t* out) {
    EXL2B_REQUIRE(d && out, "null argument");
    // down may be absent (tensor-parallel rank: gate|up on its intermediate slice, exl2b_qmlp_forward_gateup)
    EXL2B_REQUIRE(d->gate && d->up, "gate/up handles are required");
    const QMatrix *g = (const QMatrix*)d->gate, *u = (const QMatrix*)d->up, *dn = d->down ? (const QMatrix*)d->down : nullptr;
    EXL2B_REQUIRE(g->v.K == d->hidden_size && u->v.K == d->hidden_size && (!dn || dn->v.N == d->hidden_size), "mlp matrices have wrong shape");
    EXL2B_REQUIRE(g->v.N == d->intermediate_size && u->v.N == d->intermediate_size && (!dn || dn->v.K == d->intermediate_size),
                  "mlp intermediate size mismatch");
    EXL2B_REQUIRE(g->device == u->device && (!dn || g->device == dn->device), "handles on different devices");
    const QMatrix* gu[2] = {g, u};
    const bool i8 = gemv_i8_fusable(gu, 2);
    half* norm_p = nullptr;
    int rc = block_norm_copy(g, d->layernorm, i8, &norm_p);
    if (rc) return rc;
    QMlp* m = new QMlp{*d, g->device, i8, nullptr, norm_p};
    *out = (exl2b_qmlp_t)m;
    return 0;
}

extern "C" int exl2b_qmlp_destroy(exl2b_qmlp_t h) {
    QMlp* m = (QMlp*)h;
    if (m && (m->up_scratch || m->norm_p)) {
        cudaSetDevice(m->device);
        if (m->up_scratch) cudaFree(m->up_scratch);
        if (m->norm_p) cudaFree(m->norm_p);
    }
    delete m;
    return 0;
}

extern "C" int exl2b_qmlp_forward(exl2b_qmlp_t h, uint16_t* x, int rows, uint16_t* temp_a, uint16_t* temp_b, int input_prepared,
                                  const exl2b_chain_t* next, const uint64_t* ids, int num_ids, exl2b_stream_t stream_) {
    QMlp* m = (QMlp*)h;
    EXL2B_REQUIRE(m && x && temp_a && (ids || num_ids == 0), "null argument");
    EXL2B_REQUIRE(m->d.down, "this MLP handle was created without down_proj");
    LoraParams gu = {}, dn = {};
    int rc = lora_stack(m->loras, ids, num_ids, MLP_STAGES[0], 2, gu);
    if (!rc) rc = lora_stack(m->loras, ids, num_ids, MLP_STAGES[1], 1, dn);
    if (rc) return rc;
    EXL2B_CUDA(cudaSetDevice(m->device));
    cudaStream_t stream = (cudaStream_t)stream_;
    if (gu.nseg == 0 && dn.nseg == 0) return mlp_stages(m, x, rows, temp_a, temp_b, input_prepared, next, stream);
    if (!is_chained(input_prepared, next)) return mlp_lora(m, x, rows, temp_a, temp_b, gu, dn, stream);
    const QMatrix* gud[3] = {(const QMatrix*)m->d.gate, (const QMatrix*)m->d.up, (const QMatrix*)m->d.down};
    rc = lora_chain_rule(rows, row_path(rows, gud, 3, m->i8_gu && gud[2]->v.layout == LAYOUT_TC, true));
    if (rc) return rc;
    return mlp_row(m, x, temp_a, temp_b, input_prepared, next, &gu, &dn, stream);
}

// first half of the MLP only: temp_a[rows, intermediate] = act(norm(x) @ gate) * (norm(x) @ up)   (x is not modified)
extern "C" int exl2b_qmlp_forward_gateup(exl2b_qmlp_t h, const uint16_t* x, int rows, uint16_t* temp_a, exl2b_stream_t stream_) {
    QMlp* m = (QMlp*)h;
    EXL2B_REQUIRE(m && x && temp_a, "null argument");
    EXL2B_CUDA(cudaSetDevice(m->device));
    const QMatrix* gu[2] = {(const QMatrix*)m->d.gate, (const QMatrix*)m->d.up};
    return gate_up_stage(m, row_path(rows, gu, 2, m->i8_gu, false), x, rows, temp_a, nullptr, true, (cudaStream_t)stream_);
}

// gemm_half_q_half whose input was prepared by a chained producer (lm_head after the last MLP: the final RMSNorm is the
// producer's scatter scale + this launch's deferred 1/rms)
extern "C" int exl2b_gemm_half_q_half_prepared(exl2b_qmatrix_t h, uint16_t* c, int ldc, int m, int clear, int has_norm,
                                               float norm_eps, exl2b_stream_t stream) {
    QMatrix* q = (QMatrix*)h;
    EXL2B_REQUIRE(q && c, "null argument");
    EXL2B_REQUIRE(ldc >= q->v.N, "leading dimension too small");
    EXL2B_CUDA(cudaSetDevice(q->device));
    GemvMat mt = make_mat(q, nullptr, q->v.K, (half*)c, ldc, clear ? 1 : 0);
    EXL2B_REQUIRE(gemv_supports_extras(&mt, 1, m, true), CHAIN_RULE, GEMV_MAX_CHAIN_ROWS);
    GemvExtras ex = {};
    const QMatrix* qc = q;
    int rc = chain_in(ex, &mt, &qc, 1, has_norm != 0, m);
    if (rc) return rc;
    return gemv_launch(q->device, (cudaStream_t)stream, &mt, 1, m, nullptr, norm_eps, EPI_STORE, &ex);
}

// rms_norm + gemm_half_q_half on ONE row as a single launch (final norm + lm_head of a decode step; the reference runs
// rms_norm_cuda then gemm_half_q_half_cuda, exllamav2/model.py:1036-1044 -> rmsnorm.py:141, linear.py:366).
// x == NULL: the row was left in this matrix's stored-row order by a chained producer launch.
extern "C" int exl2b_gemm_half_q_half_norm(exl2b_qmatrix_t h, const uint16_t* x, const uint16_t* norm_w, float norm_eps,
                                           uint16_t* c, int clear, exl2b_stream_t stream) {
    QMatrix* q = (QMatrix*)h;
    EXL2B_REQUIRE(q && norm_w && c, "null argument");
    EXL2B_REQUIRE(q->v.layout == LAYOUT_TC, "matrix is not in the default layout");
    EXL2B_CUDA(cudaSetDevice(q->device));
    const I8Out o = {q, (half*)c, clear ? 1 : 0};
    I8Input in = {(const half*)x, nullptr, (const half*)norm_w, norm_eps, I8_RMSNORM, 0};
    if (!x) {
        EXL2B_REQUIRE(q->xp_buf, "no input row given and no chained producer has written this matrix's input row");
        in.x = q->xp_buf;
        in.x_permuted = 1;
    }
    return gemv_i8_launch(q->device, (cudaStream_t)stream, &o, 1, in);
}

extern "C" int exl2b_qattn_set_loras(exl2b_qattn_t h, const exl2b_lora_t* loras, int num, int* max_rank) {
    QAttn* a = (QAttn*)h;
    EXL2B_REQUIRE(a, "null argument");
    const QMatrix* ms[4] = {(const QMatrix*)a->d.q_proj, (const QMatrix*)a->d.k_proj, (const QMatrix*)a->d.v_proj,
                            (const QMatrix*)a->d.o_proj};
    int ks[4], ns[4];
    for (int p = 0; p < 4; ++p) {
        ks[p] = ms[p] ? ms[p]->v.K : -1;
        ns[p] = ms[p] ? ms[p]->v.N : -1;
    }
    return lora_take(loras, num, ks, ns, 4, ATTN_STAGES, 2, a->loras, max_rank);
}

extern "C" int exl2b_qmlp_set_loras(exl2b_qmlp_t h, const exl2b_lora_t* loras, int num, int* max_rank) {
    QMlp* m = (QMlp*)h;
    EXL2B_REQUIRE(m, "null argument");
    const QMatrix* ms[3] = {(const QMatrix*)m->d.gate, (const QMatrix*)m->d.up, (const QMatrix*)m->d.down};
    int ks[3], ns[3];
    for (int p = 0; p < 3; ++p) {
        ks[p] = ms[p] ? ms[p]->v.K : -1;
        ns[p] = ms[p] ? ms[p]->v.N : -1;
    }
    return lora_take(loras, num, ks, ns, 3, MLP_STAGES, 2, m->loras, max_rank);
}
