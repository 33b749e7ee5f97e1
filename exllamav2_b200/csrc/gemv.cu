// Dispatch of gemm_half_q_half over the row count, and the split-K workspace of the wgmma kernel.
//   1 row        -> gemv_i8.cu   (HBM-bound integer GEMV, the decode path)
//   2 .. 16 rows -> gemm_tc.cu   (packed weights unpacked into the wgmma A operand in shared memory, 8 rows per pass; chained
//                                  launches of up to 64 rows in one pass)
//   more         -> gemm_big.cu  (reconstruct window + dense tensor-core GEMM: the reference's regime above MAX_Q_GEMM_ROWS)
// Replaces gemm_half_q_half_cuda (exllamav2_ext/cuda/q_gemm.cu:201-313).
#include <algorithm>
#include <map>
#include <mutex>

#include "gemv.cuh"
#include "gemv_i8.cuh"

namespace exl2b {

int g_ctas_per_sm = 2;
int g_tc_ctas_per_sm = [] { const char* e = getenv("EXL2B_TC_CTAS"); return e ? atoi(e) : 2; }();
unsigned long long* g_dbg = nullptr;
int g_dbg_cta = 0;
int g_dbg_slot = 0;
unsigned long long* g_dbg_rec = nullptr;      // optional per-CTA records of the batch-1 GEMV: [64 launches][160 CTAs][4]

// Split-K workspace, arrival counters and the activation-operand scratch of the wgmma kernel, one set per (device, stream):
// launches on different streams (or host threads driving different streams) never share scratch.  Created on first use --
// never inside a stream capture: call once eagerly first, as model.capture() does.  The wide tiles (chained launches of 9..64
// rows) get their own workspace and scratch, created on their first launch and never moved: a graph captured before holds the
// 8-row buffers' addresses.  Both share the counters (a launch touches them only after the previous launch has completed).
struct TcWorkspace {
    float* ws = nullptr;
    unsigned int* counters = nullptr;
    half* xp = nullptr;
    size_t ws_bytes = 0, xp_bytes = 0;
    int n_counters = 0;
    float* ws_wide = nullptr;
    half* xp_wide = nullptr;
};
static std::map<std::pair<int, cudaStream_t>, TcWorkspace> g_tc_ws;
static std::mutex g_ws_mutex;

int gemv_workspace(int device, cudaStream_t stream, bool wide, float** ws, unsigned int** counters, size_t* ws_bytes, int* n_counters,
                   half** xp, size_t* xp_bytes) {
    std::lock_guard<std::mutex> lock(g_ws_mutex);
    TcWorkspace& d = g_tc_ws[{device, stream}];
    if (!d.ws) {
        d.ws_bytes = TC_WS_BYTES;
        d.n_counters = 1 << 16;
        EXL2B_CUDA(cudaMalloc(&d.ws, d.ws_bytes));
        EXL2B_CUDA(cudaMalloc(&d.counters, d.n_counters * sizeof(unsigned int)));
        EXL2B_CUDA(cudaMemset(d.counters, 0, d.n_counters * sizeof(unsigned int)));
        EXL2B_CUDA(cudaDeviceSynchronize());
    }
    if (!d.xp) {
        EXL2B_CUDA(cudaMalloc(&d.xp, TC_XP_BYTES));
        d.xp_bytes = TC_XP_BYTES;
    }
    if (wide && !d.ws_wide) {
        EXL2B_CUDA(cudaMalloc(&d.ws_wide, TC_WIDE_WS_BYTES));
        EXL2B_CUDA(cudaMalloc(&d.xp_wide, TC_WIDE_XP_BYTES));
        EXL2B_CUDA(cudaDeviceSynchronize());
    }
    *ws = wide ? d.ws_wide : d.ws;
    *counters = d.counters;
    *ws_bytes = wide ? TC_WIDE_WS_BYTES : d.ws_bytes;
    *n_counters = d.n_counters;
    *xp = wide ? d.xp_wide : d.xp;
    *xp_bytes = wide ? TC_WIDE_XP_BYTES : d.xp_bytes;
    return 0;
}

int gemm_tc_launch(int device, cudaStream_t stream, GemvMat* mats, int nm, int M, const half* norm_w, float norm_eps, int epilogue,
                   const GemvExtras* ex);

bool gemm_tc_supported(const QMatView& v);
bool gemv_supports_extras(const GemvMat* mats, int nm, int M, bool chained) {
    for (int i = 0; i < nm; ++i)
        if (mats[i].w.layout != LAYOUT_TC || !gemm_tc_supported(mats[i].w)) return false;
    return M >= 1 && M <= (chained ? GEMV_MAX_CHAIN_ROWS : GEMV_MTOK);
}

int gemv_launch(int device, cudaStream_t stream, GemvMat* mats, int nm, int M, const half* norm_w, float norm_eps,
                int epilogue, const GemvExtras* ex) {
    EXL2B_REQUIRE(nm >= 1 && nm <= GEMV_MAX_MATS, "bad matrix count %d", nm);
    EXL2B_REQUIRE(device >= 0 && device < 64, "bad device %d", device);
    if (M <= 0) return 0;
    for (int i = 0; i < nm; ++i) EXL2B_REQUIRE(mats[i].w.layout == LAYOUT_TC, "matrix is not in the default (LAYOUT_TC) layout");
    return gemm_tc_launch(device, stream, mats, nm, M, norm_w, norm_eps, epilogue, ex);
}

// The wgmma kernel stages one quantisation group of a 32-column block per ring slot: at most 4 slabs (128 rows, the size of
// its activation stage) and 4 KB of weights.  Groups of 256+ rows (EXL2 g256+, GPTQ g256+, ungrouped GPTQ) do not fit; such
// matrices take the dense path for every row count above one.
bool gemm_tc_supported(const QMatView& v) {
    for (int r = 0; r < v.num_regions; ++r)
        if (v.reg[r].spg_log2 > 2 || (1 << v.reg[r].spg_log2) * block_bytes(v.reg[r].bits) > 4096) return false;
    return true;
}

RowPath row_path(int rows, const QMatrix* const* qs, int n, bool i8_fusable, bool chained) {
    if (rows == 1 && i8_fusable && gemv_i8_enabled()) return ROW_I8;
    if (chained) return ROW_TC;
    bool staged = true;
    for (int i = 0; i < n; ++i) staged = staged && gemm_tc_supported(qs[i]->v);
    return (rows > GEMM_BIG_MIN_ROWS || !staged) && gemm_big_available() ? ROW_DENSE : ROW_TC;
}

}  // namespace exl2b

using namespace exl2b;

extern "C" int exl2b_qmatrix_tc_supported(exl2b_qmatrix_t h, int* supported) {
    const QMatrix* q = (const QMatrix*)h;
    EXL2B_REQUIRE(q && supported, "null argument");
    *supported = q->v.layout == LAYOUT_TC && gemm_tc_supported(q->v) ? 1 : 0;
    return 0;
}

extern "C" int exl2b_gemm_half_q_half(exl2b_qmatrix_t h, const uint16_t* a, int lda, uint16_t* c, int ldc, int m,
                                      int clear, int force_cuda, exl2b_stream_t stream) {
    (void)force_cuda;
    QMatrix* q = (QMatrix*)h;
    EXL2B_REQUIRE(q && a && c, "null argument");
    EXL2B_REQUIRE(lda >= q->v.K && ldc >= q->v.N, "leading dimensions too small");
    EXL2B_CUDA(cudaSetDevice(q->device));
    const QMatrix* qs = q;
    RowPath path = row_path(m, &qs, 1, q->v.layout == LAYOUT_TC, false);
    if (path == ROW_I8) {        // decode row: the HBM-bound integer GEMV (gemv_i8.cu)
        const I8Out o = {q, (half*)c, clear ? 1 : 0};
        const I8Input in = {(const half*)a, nullptr, nullptr, 0.f, I8_PLAIN};
        return gemv_i8_launch(q->device, (cudaStream_t)stream, &o, 1, in);
    }
    // 9..16 rows would be two 8-row passes of the wgmma kernel, each re-reading the weights: on matrices up to ~20 M weights
    // the dense path takes them (measured for single matrices; the blocks do not apply it)
    const bool small_two_pass = m > GEMV_MTOK && (long long)q->v.K * q->v.N <= 20ll * 1000 * 1000;
    if (path == ROW_TC && small_two_pass && gemm_big_available()) path = ROW_DENSE;
    if (path == ROW_DENSE)       // prefill rows: reconstruct + tensor-core GEMM (q_gemm.cu:233-266)
        return gemm_big_launch(q, (const half*)a, lda, (half*)c, ldc, m, clear ? 1 : 0, (cudaStream_t)stream);
    GemvMat mt = {};
    mt.w = q->v;
    mt.x = (const half*)a;
    mt.ldx = lda;
    mt.c = (half*)c;
    mt.ldc = ldc;
    mt.clear = clear ? 1 : 0;
    return gemv_launch(q->device, (cudaStream_t)stream, &mt, 1, m, nullptr, 0.f, EPI_STORE);
}

extern "C" int exl2b_gemm_half_q_half_host(exl2b_qmatrix_t h, const uint16_t* a_host, uint16_t* c_host, int m,
                                           exl2b_stream_t stream_) {
    QMatrix* q = (QMatrix*)h;
    EXL2B_REQUIRE(q && a_host && c_host && m > 0, "bad argument");
    cudaStream_t stream = (cudaStream_t)stream_;
    EXL2B_CUDA(cudaSetDevice(q->device));
    const size_t ab = (size_t)m * q->v.K * 2, cb = (size_t)m * q->v.N * 2;
    uint16_t *da = nullptr, *dc = nullptr;
    EXL2B_CUDA(cudaMallocAsync(&da, ab, stream));
    EXL2B_CUDA(cudaMallocAsync(&dc, cb, stream));
    EXL2B_CUDA(cudaMemcpyAsync(da, a_host, ab, cudaMemcpyHostToDevice, stream));
    int rc = exl2b_gemm_half_q_half(h, da, q->v.K, dc, q->v.N, m, 1, 0, stream_);
    if (rc == 0) {
        EXL2B_CUDA(cudaMemcpyAsync(c_host, dc, cb, cudaMemcpyDeviceToHost, stream));
    }
    cudaFreeAsync(da, stream);
    cudaFreeAsync(dc, stream);
    EXL2B_CUDA(cudaStreamSynchronize(stream));
    return rc;
}

// ---- tuning / diagnostics hooks (not part of the reference surface) ---------------------------------------------------
extern "C" int exl2b_debug_set(int ctas_per_sm, unsigned long long* stamps, int cta) {
    if (ctas_per_sm > 0) { exl2b::g_ctas_per_sm = ctas_per_sm; exl2b::g_tc_ctas_per_sm = ctas_per_sm; }
    exl2b::g_dbg = stamps;
    exl2b::g_dbg_cta = cta;
    exl2b::g_dbg_slot = 0;
    return 0;
}
extern "C" int exl2b_debug_set_records(unsigned long long* records) {
    exl2b::g_dbg_rec = records;
    return 0;
}

namespace exl2b {
int attn_scratch_query(int device, cudaStream_t stream, int kind, void** ptr, size_t* bytes);
}
extern "C" int exl2b_debug_scratch(int device, exl2b_stream_t stream, int kind, void** ptr, size_t* bytes) {
    EXL2B_REQUIRE(ptr && bytes && device >= 0 && device < 64, "bad argument");
    EXL2B_REQUIRE(kind >= EXL2B_SCRATCH_ATTN_WS && kind <= EXL2B_SCRATCH_TC_XP_WIDE, "unknown scratch kind %d", kind);
    if (kind == EXL2B_SCRATCH_ATTN_WS || kind == EXL2B_SCRATCH_ATTN_CNT)
        return attn_scratch_query(device, (cudaStream_t)stream, kind, ptr, bytes);
    std::lock_guard<std::mutex> lock(g_ws_mutex);
    *ptr = nullptr;
    *bytes = 0;
    const auto it = g_tc_ws.find({device, (cudaStream_t)stream});
    if (it == g_tc_ws.end()) return 0;
    const TcWorkspace& d = it->second;
    if (kind == EXL2B_SCRATCH_TC_WS) { *ptr = d.ws; *bytes = d.ws_bytes; }
    if (kind == EXL2B_SCRATCH_TC_CNT) { *ptr = d.counters; *bytes = (size_t)d.n_counters * sizeof(unsigned int); }
    if (kind == EXL2B_SCRATCH_TC_XP) { *ptr = d.xp; *bytes = d.xp_bytes; }
    if (kind == EXL2B_SCRATCH_TC_WS_WIDE && d.ws_wide) { *ptr = d.ws_wide; *bytes = TC_WIDE_WS_BYTES; }
    if (kind == EXL2B_SCRATCH_TC_XP_WIDE && d.xp_wide) { *ptr = d.xp_wide; *bytes = TC_WIDE_XP_BYTES; }
    return 0;
}
