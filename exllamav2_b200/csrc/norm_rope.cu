// Stand-alone RMSNorm, RoPE and act*mul kernels behind the reference's rms_norm / rope_ / act_mul bindings.
// (On the fused decode path RMSNorm lives in the GEMV prologue and silu*mul in its epilogue; these kernels serve
// the direct ext_c.rms_norm / ext_c.rope_ calls and batched rows.)
#include "common.cuh"

namespace exl2b {

// ---- RMSNorm: cuda/rms_norm.cu:34-175.  One 256-thread CTA per row, 128-bit loads, fp32 statistics. -------------
__global__ void __launch_bounds__(256) rms_norm_kernel(const half* __restrict__ x, const half* __restrict__ w,
                                                       half* __restrict__ y, float eps, int dim) {
    griddep_launch_dependents();
    griddep_wait();
    const int row = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const half* xr = x + (size_t)row * dim;
    half* yr = y + (size_t)row * dim;
    __shared__ float sums[8];
    float sum = 0.f;
    for (int k = tid * 8; k < dim; k += 256 * 8) {
        if (k + 8 <= dim) {
            const uint4 v = *reinterpret_cast<const uint4*>(xr + k);
            const half2* h = reinterpret_cast<const half2*>(&v);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                float f0 = fmaxf(-65504.f, fminf(__low2float(h[i]), 65504.f));
                float f1 = fmaxf(-65504.f, fminf(__high2float(h[i]), 65504.f));
                sum = fmaf(f0, f0, sum);
                sum = fmaf(f1, f1, sum);
            }
        } else {
            for (int i = k; i < dim; ++i) {
                float f = fmaxf(-65504.f, fminf(__half2float(xr[i]), 65504.f));
                sum = fmaf(f, f, sum);
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) sums[warp] = sum;
    __syncthreads();
    sum = (lane < 8) ? sums[lane] : 0.f;
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    sum = __shfl_sync(0xffffffffu, sum, 0);
    const float r = rsqrtf(sum * (1.0f / (float)dim) + eps);
    for (int k = tid * 8; k < dim; k += 256 * 8) {
        if (k + 8 <= dim) {
            const uint4 v = *reinterpret_cast<const uint4*>(xr + k);
            const uint4 wv = *reinterpret_cast<const uint4*>(w + k);
            const half2* h = reinterpret_cast<const half2*>(&v);
            const half2* wh = reinterpret_cast<const half2*>(&wv);
            uint4 o4;
            half2* oh = reinterpret_cast<half2*>(&o4);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                float f0 = fmaxf(-65504.f, fminf(__low2float(h[i]), 65504.f));
                float f1 = fmaxf(-65504.f, fminf(__high2float(h[i]), 65504.f));
                oh[i] = __halves2half2(__float2half_rn(f0 * __low2float(wh[i]) * r), __float2half_rn(f1 * __high2float(wh[i]) * r));
            }
            *reinterpret_cast<uint4*>(yr + k) = o4;
        } else {
            for (int i = k; i < dim; ++i) {
                float f = fmaxf(-65504.f, fminf(__half2float(xr[i]), 65504.f));
                yr[i] = __float2half_rn(f * __half2float(w[i]) * r);
            }
        }
    }
}

// ---- RoPE: cuda/rope.cu:10-123.  One thread per half2 pair-column; same fp16 op order as the reference. ----------
__global__ void rope_kernel(half* __restrict__ x, const half* __restrict__ sin, const half* __restrict__ cos,
                            int rows_per_batch, int head_dim, int num_heads, int past_len,
                            const int32_t* __restrict__ past_lens, int neox, int sincos_size) {
    griddep_launch_dependents();
    griddep_wait();
    const int cols = neox ? (sincos_size / 2) / 2 : sincos_size / 2;       // half2 columns handled per row
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= rows_per_batch * cols) return;
    const int row = idx / cols, column = (idx - row * cols) * 2;
    const int b = blockIdx.y;
    if (past_len == -1) {
        past_len = max(past_lens[b], 0);
    } else if (past_lens) {
        past_len += past_lens[b];
    }
    const int sincos_row = max(past_len + row / num_heads, 0);
    half* xr = x + ((size_t)b * rows_per_batch + row) * head_dim;
    const half* sr = sin + (size_t)sincos_row * sincos_size;
    const half* cr = cos + (size_t)sincos_row * sincos_size;
    if (neox) {
        const int half_dim = sincos_size / 2;
        const half2 c2 = *reinterpret_cast<const half2*>(cr + column);
        const half2 s2 = *reinterpret_cast<const half2*>(sr + column);
        const half2 ns2 = __hneg2(s2);
        half2 l = *reinterpret_cast<half2*>(xr + column);
        half2 r = *reinterpret_cast<half2*>(xr + column + half_dim);
        const half2 ls = __hmul2(r, ns2);
        const half2 rs = __hmul2(l, s2);
        l = __hfma2(l, c2, ls);
        r = __hfma2(r, c2, rs);
        *reinterpret_cast<half2*>(xr + column) = l;
        *reinterpret_cast<half2*>(xr + column + half_dim) = r;
    } else {
        const half2 c01 = *reinterpret_cast<const half2*>(cr + column);
        half2 s01 = *reinterpret_cast<const half2*>(sr + column);
        uint32_t sb = *reinterpret_cast<uint32_t*>(&s01) ^ (1u << 15);      // (-sin[i], +sin[i+1])
        s01 = *reinterpret_cast<half2*>(&sb);
        const half2 x01 = *reinterpret_cast<half2*>(xr + column);
        const half2 x10 = __lowhigh2highlow(x01);
        half2 r = __hmul2(x01, c01);
        r = __hfma2(x10, s01, r);
        *reinterpret_cast<half2*>(xr + column) = r;
    }
}

// ---- act * mul: cuda/q_mlp_activation.cuh:54-130 -----------------------------------------------------------------
__global__ void act_mul_kernel(half* __restrict__ x, const half* __restrict__ y, size_t n2, int gelu) {
    griddep_launch_dependents();
    griddep_wait();
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n2) return;
    half2 xv = reinterpret_cast<half2*>(x)[i];
    const half2 yv = reinterpret_cast<const half2*>(y)[i];
    xv = gelu ? __halves2half2(gelu1(__low2half(xv)), gelu1(__high2half(xv))) : silu2(xv);
    reinterpret_cast<half2*>(x)[i] = __hmul2(xv, yv);
}

int rope_launch(cudaStream_t stream, half* x, const half* sin, const half* cos, int batch, int rows_per_batch, int head_dim,
                int num_heads, int past_len, const int32_t* past_lens, int neox, int sincos_size) {
    const int cols = neox ? (sincos_size / 2) / 2 : sincos_size / 2;
    const long total = (long)rows_per_batch * cols;
    if (total <= 0 || batch <= 0) return 0;
    dim3 grid((unsigned)((total + 127) / 128), batch);
    EXL2B_CUDA(launch_pdl(rope_kernel, grid, dim3(128), 0, stream, x, sin, cos, rows_per_batch, head_dim, num_heads, past_len,
                          past_lens, neox, sincos_size));
    return 0;
}

}  // namespace exl2b

using namespace exl2b;

extern "C" int exl2b_rms_norm(const uint16_t* x, const uint16_t* w, uint16_t* y, float eps, int rows, int dim,
                              exl2b_stream_t stream) {
    EXL2B_REQUIRE(x && w && y && dim > 0, "bad argument");
    EXL2B_REQUIRE(dim % 8 == 0, "rms_norm: dim %d must be a multiple of 8", dim);
    if (rows <= 0) return 0;
    EXL2B_CUDA(launch_pdl(rms_norm_kernel, dim3(rows), dim3(256), 0, (cudaStream_t)stream, (const half*)x, (const half*)w,
                          (half*)y, eps, dim));
    return 0;
}

extern "C" int exl2b_rope(uint16_t* x, const uint16_t* sin, const uint16_t* cos, int batch, int rows_per_batch,
                          int head_dim, int num_heads, int past_len, const int32_t* past_lens, int neox,
                          int sincos_size, exl2b_stream_t stream) {
    EXL2B_REQUIRE(x && sin && cos, "bad argument");
    EXL2B_REQUIRE(head_dim % 2 == 0 && sincos_size % 4 == 0, "rope: bad head_dim/sincos_size");
    return rope_launch((cudaStream_t)stream, (half*)x, (const half*)sin, (const half*)cos, batch, rows_per_batch, head_dim,
                       num_heads, past_len, past_lens, neox, sincos_size);
}

extern "C" int exl2b_act_mul(uint16_t* x, const uint16_t* y, int rows, int width, int act_gelu, exl2b_stream_t stream) {
    EXL2B_REQUIRE(x && y && width % 2 == 0, "bad argument");
    const size_t n2 = (size_t)rows * width / 2;
    if (!n2) return 0;
    EXL2B_CUDA(launch_pdl(act_mul_kernel, dim3((unsigned)((n2 + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, (half*)x,
                          (const half*)y, n2, act_gelu));
    return 0;
}
