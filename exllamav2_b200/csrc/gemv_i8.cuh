// Batch-1 dequant-GEMV on the integer dot-product pipe (gemv_i8.cu): host interface.
#pragma once
#include "qmatrix.cuh"

namespace exl2b {

constexpr int I8_MAX_MATS = 3;

// What the kernel's prologue does to the input row before it is quantised to 16-bit integers:
enum I8Mode : int {
    I8_PLAIN = 0,      // a = x
    I8_RMSNORM = 1,    // a = x * w * rsqrt(mean(x^2) + eps)      rms_norm_kernel, cuda/rms_norm.cu:55-143 (1/rms applied to the fp32 sum)
    I8_SILU_MUL = 2,   // a = half(half(silu(x)) * x2)             act_mul_kernel, cuda/q_mlp_activation.cuh:54-100 (same fp16 op order)
    I8_GELU_MUL = 3,
};

struct I8Input {
    const half* x;        // fp16 [K]
    const half* x2;       // fp16 [K] (I8_*_MUL) or NULL
    const half* norm_w;   // fp16 [K] (I8_RMSNORM) or NULL, ORIGINAL feature order
    float norm_eps;
    int mode;
    int x_permuted;       // x / x2 are already in the matrices' stored-row order (written by a producer launch's c_perm)
    const half* norm_wp;  // norm_w in the matrices' stored-row order (permuted_norm_copy, owned by a block handle), or NULL:
                          //   the kernel gathers norm_w through the permutation itself
};

struct I8Out {
    const QMatrix* q;
    half* c;                       // fp16 [N]
    int clear;                     // 1: c = acc (+bias); 0: c += acc (+bias)   (residual add, cuda/q_attn.cu:333)
    half* c_perm;                  // optional second copy of the NEW c, scattered to c_perm[out_invperm[n]] -- the row order of
    const uint16_t* out_invperm;   //   the matrix that consumes it next (then that launch reads it contiguously: x_permuted)
};

// One launch over `nm` matrices that share K, the input row and the row permutation.  M = 1 only.
int gemv_i8_launch(int device, cudaStream_t stream, const I8Out* outs, int nm, const I8Input& in);
// same K / same permutation contents / LAYOUT_TC?  (host check, synchronises once; call at block-creation time)
bool gemv_i8_fusable(const QMatrix* const* qs, int nm);
// a new device copy of norm_w[perm[k]] in q's stored-row order (cudaFree it); synchronises, never call inside a capture
int permuted_norm_copy(const QMatrix* q, const half* norm_w, half** out);
// EXL2B_GEMV=tc in the environment routes single rows through the wgmma kernel (gemm_tc.cu) instead (A/B comparisons)
bool gemv_i8_enabled();

}  // namespace exl2b
