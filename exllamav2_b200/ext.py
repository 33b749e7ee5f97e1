"""`exllamav2_ext`-compatible operator surface over libexl2b200.so (ctypes, C ABI in include/exl2_b200.h).

Every public function below has the NAME, ARGUMENT ORDER and meaning of the reference pybind binding it replaces
(exllamav2/exllamav2_ext/ext_bindings.cpp:27-138), so exllamav2/{linear,attn,mlp,cache,rmsnorm}.py call it
unchanged when this module is importable as `exllamav2_ext` (see INTEGRATION.md; `install_as_exllamav2_ext()`).
torch is used only for device memory / the current stream -- all arithmetic is in the CUDA library.

The product path fails loudly: importing this module without the built library, or calling an op on CPU tensors,
raises.  There is no CPU or PyTorch fallback.
"""
from __future__ import annotations

import ctypes
import os
import sys
from ctypes import POINTER, Structure, c_char_p, c_float, c_int, c_int16, c_int32, c_uint64, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libexl2b200.so")

if not os.path.exists(_LIB_PATH):
    raise ImportError(
        f"{_LIB_PATH} is missing: build it with `python -m exllamav2_b200.build` (nvcc, sm_90a). "
        "exllamav2_b200 has no CPU fallback.")

lib = ctypes.CDLL(_LIB_PATH)


class _QMatrixDesc(Structure):
    _fields_ = [
        ("device", c_int), ("height", c_int), ("width", c_int), ("groups", c_int),
        ("q_weight", c_void_p), ("q_perm", c_void_p), ("q_invperm", c_void_p),
        ("q_scale", c_void_p), ("q_scale_max", c_void_p), ("q_groups", c_void_p), ("q_weight_rows", c_int),
        ("gptq_qzeros", c_void_p), ("gptq_scales", c_void_p), ("gptq_g_idx", c_void_p), ("bias", c_void_p),
    ]


class _QAttnDesc(Structure):
    _fields_ = [
        ("layernorm", c_void_p), ("norm_epsilon", c_float),
        ("q_proj", c_void_p), ("k_proj", c_void_p), ("v_proj", c_void_p), ("o_proj", c_void_p),
        ("hidden_size", c_int), ("num_heads", c_int), ("num_kv_heads", c_int), ("head_dim", c_int),
        ("has_residual", c_int), ("rope_style", c_int), ("sincos_size", c_int),
    ]


class _QMlpDesc(Structure):
    _fields_ = [
        ("layernorm", c_void_p), ("norm_epsilon", c_float),
        ("gate", c_void_p), ("up", c_void_p), ("down", c_void_p),
        ("hidden_size", c_int), ("intermediate_size", c_int), ("act_gelu", c_int), ("has_residual", c_int),
    ]


def _sig(name, restype, *argtypes):
    f = getattr(lib, name)
    f.restype = restype
    f.argtypes = list(argtypes)
    return f


_sig("exl2b_last_error", c_char_p)
_sig("exl2b_version", c_int)
_sig("exl2b_launch_count", c_uint64)
_sig("exl2b_row_gemv_i8", c_int)
_sig("exl2b_qmatrix_create", c_int, POINTER(_QMatrixDesc), c_void_p, POINTER(c_void_p))
_sig("exl2b_qmatrix_destroy", c_int, c_void_p)
_sig("exl2b_qmatrix_info", c_int, c_void_p, POINTER(c_int), POINTER(c_int), POINTER(c_int), POINTER(c_int), POINTER(c_uint64))
_sig("exl2b_qmatrix_tc_supported", c_int, c_void_p, POINTER(c_int))
_sig("exl2b_reconstruct", c_int, c_void_p, c_void_p, c_void_p)
_sig("exl2b_gemm_half_q_half", c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p)
_sig("exl2b_gemm_half_q_half_norm", c_int, c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_int, c_void_p)
_sig("exl2b_gemm_half_q_half_host", c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p)
_sig("exl2b_make_group_map", c_int, POINTER(c_int16), c_int, c_int, POINTER(c_int16), c_int, POINTER(c_int))
_sig("exl2b_rms_norm", c_int, c_void_p, c_void_p, c_void_p, c_float, c_int, c_int, c_void_p)
_sig("exl2b_rope", c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p)
_sig("exl2b_act_mul", c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p)
_KV_ARGS = (c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
            c_void_p, c_void_p, c_int, c_int, c_void_p)
_sig("exl2b_fp16_to_q_kv", c_int, *_KV_ARGS)
_sig("exl2b_q_to_fp16_kv", c_int, *_KV_ARGS)
_sig("exl2b_qattn_create", c_int, POINTER(_QAttnDesc), POINTER(c_void_p))
_sig("exl2b_qattn_destroy", c_int, c_void_p)
_sig("exl2b_qmlp_create", c_int, POINTER(_QMlpDesc), POINTER(c_void_p))
_sig("exl2b_qmlp_destroy", c_int, c_void_p)
_sig("exl2b_qmlp_forward_gateup", c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p)
_sig("exl2b_paged_attn_decode_q", c_int, *([c_void_p] * 10 + [c_int] * 7 + [c_float, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]))
_sig("exl2b_paged_attn_prefill_q", c_int, *([c_void_p] * 10 + [c_int] * 7 + [c_float, c_int, c_void_p]))
_sig("exl2b_paged_attn_status", c_int, c_int, POINTER(c_int))
_sig("exl2b_paged_attn_clear_status", c_int, c_int)
_sig("exl2b_debug_scratch", c_int, c_int, c_void_p, c_int, POINTER(c_void_p), POINTER(ctypes.c_size_t))


class _Chain(Structure):
    _fields_ = [("consumers", c_void_p * 3), ("num_consumers", c_int), ("norm_weight", c_void_p)]


# the block forwards (include/exl2_b200.h "block forwards"): ..., input_prepared, next, ids, num_ids, stream
_sig("exl2b_qattn_forward_1", c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
     c_void_p, c_void_p, c_int, POINTER(c_uint64), c_int, c_void_p)
_sig("exl2b_qattn_forward_2", c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, POINTER(_Chain), POINTER(c_uint64), c_int,
     c_void_p)
_sig("exl2b_qmlp_forward", c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, POINTER(_Chain), POINTER(c_uint64), c_int,
     c_void_p)
_sig("exl2b_gemm_half_q_half_prepared", c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p)


class _Lora(Structure):
    _fields_ = [("id", c_uint64), ("a", c_void_p * 4), ("b", c_void_p * 4), ("rank", c_int * 4), ("a_rows", c_int * 4),
                ("b_cols", c_int * 4)]


_sig("exl2b_qattn_set_loras", c_int, c_void_p, POINTER(_Lora), c_int, POINTER(c_int))
_sig("exl2b_qmlp_set_loras", c_int, c_void_p, POINTER(_Lora), c_int, POINTER(c_int))
_sig("exl2b_lora_stack", c_int, POINTER(c_int), c_int, c_int, POINTER(c_int), POINTER(c_int), POINTER(c_int), POINTER(c_int),
     POINTER(c_int))

# Dummy tensor standing for None/NULL (ext.py:296 of the reference)
none_tensor = torch.empty((1, 1), device="meta")


def _check(rc: int):
    if rc != 0:
        raise RuntimeError(lib.exl2b_last_error().decode())


def _p(t: torch.Tensor | None):
    """device pointer or NULL for the meta-device `none_tensor`."""
    if t is None or t.is_meta:
        return None
    return t.data_ptr()


def _cuda(t: torch.Tensor, what: str):
    if not t.is_cuda:
        raise RuntimeError(f"{what} must be a CUDA tensor: exllamav2_b200 has no CPU path")
    return t


def _dtype(t: torch.Tensor, dt, what: str):
    if t.dtype != dt:
        raise RuntimeError(f"{what} is incorrect datatype, must be {dt}")     # TORCH_CHECK_DTYPE, cpp/util.h:34


def _stream(t: torch.Tensor):
    return torch.cuda.current_stream(t.device).cuda_stream


def launch_count() -> int:
    return int(lib.exl2b_launch_count())


def row_gemv_i8() -> bool:
    """True if single rows run on the integer GEMV (csrc/gemv_i8.cu), False if on the wgmma kernel (EXL2B_GEMV=tc at load)."""
    return bool(lib.exl2b_row_gemv_i8())


# ---------------------------------------------------------------------------------------------------------------
# QMatrix
# ---------------------------------------------------------------------------------------------------------------

def make_q_matrix(q_weight, q_perm, q_invperm, q_scale, q_scale_max, q_groups, q_group_map, gptq_qzeros, gptq_scales,
                  gptq_g_idx, bias, temp_dq, max_dq_rows: int) -> int:
    """ext_qmatrix.cpp:21-111.  Same 13 arguments; temp_dq / max_dq_rows / q_group_map are accepted and unused
    (no reconstruct+cuBLAS detour, the group table is rebuilt from q_groups)."""
    _cuda(q_weight, "q_weight")
    _dtype(q_weight, torch.int32, "q_weight")
    d = _QMatrixDesc()
    d.device = q_weight.device.index or 0
    d.width = q_weight.shape[1]
    d.q_weight = _p(q_weight)
    d.q_weight_rows = q_weight.shape[0]
    d.q_perm = _p(q_perm)
    d.q_invperm = _p(q_invperm)
    d.bias = _p(bias)
    if not q_scale.is_meta:
        _dtype(q_scale, torch.int32, "q_scale")
        _dtype(q_scale_max, torch.float16, "q_scale_max")
        _dtype(q_groups, torch.int16, "q_groups")
        if q_weight.shape[1] != q_scale.shape[1] * 8:
            raise RuntimeError("q_weight and q_scale have incompatible shapes")      # TORCH_CHECK_SHAPES(...,8)
        d.groups = q_scale.shape[0]
        if not q_perm.is_meta:
            _dtype(q_perm, torch.int16, "q_perm")
            d.height = q_perm.shape[0]
        elif not q_group_map.is_meta:
            d.height = q_group_map.shape[0] // 2
        else:
            raise RuntimeError("EXL2 matrix needs q_perm or q_group_map to define its height")
        d.q_scale = _p(q_scale)
        d.q_scale_max = _p(q_scale_max)
        d.q_groups = _p(q_groups)
        keep = None
    else:
        _dtype(gptq_qzeros, torch.int32, "gptq_qzeros")
        _dtype(gptq_scales, torch.float16, "gptq_scales")
        if q_weight.shape[1] != gptq_qzeros.shape[1] * 8 or q_weight.shape[1] != gptq_scales.shape[1]:
            raise RuntimeError("qweight, qzeros and scales have incompatible shapes")
        d.groups = gptq_qzeros.shape[0]
        d.height = q_weight.shape[0] * 8
        d.gptq_qzeros = _p(gptq_qzeros)
        d.gptq_scales = _p(gptq_scales)
        keep = None
        if not gptq_g_idx.is_meta:
            keep = gptq_g_idx.to(device="cpu", dtype=torch.int32).contiguous()
            d.gptq_g_idx = keep.data_ptr()
    out = c_void_p()
    with torch.cuda.device(q_weight.device):
        _check(lib.exl2b_qmatrix_create(ctypes.byref(d), _stream(q_weight), ctypes.byref(out)))
    del keep
    return out.value


def free_q_matrix(handle: int):
    _check(lib.exl2b_qmatrix_destroy(handle))


def q_matrix_info(handle: int) -> dict:
    h, w, g, gq, pb = c_int(), c_int(), c_int(), c_int(), c_uint64()
    _check(lib.exl2b_qmatrix_info(handle, ctypes.byref(h), ctypes.byref(w), ctypes.byref(g), ctypes.byref(gq), ctypes.byref(pb)))
    return {"height": h.value, "width": w.value, "groups": g.value, "is_gptq": bool(gq.value), "packed_bytes": pb.value}


def qmatrix_tc_supported(handle: int) -> bool:
    """True if the 2..16-row kernel can stage this matrix's quantisation groups, so chained launches above one row can use it
    (include/exl2_b200.h exl2b_qmatrix_tc_supported).  Otherwise the blocks run it on the dense path above one row."""
    s = c_int()
    _check(lib.exl2b_qmatrix_tc_supported(handle, ctypes.byref(s)))
    return bool(s.value)


def reconstruct(q_handle: int, output: torch.Tensor):
    """ext_qmatrix.cpp:196-210"""
    _cuda(output, "output")
    _dtype(output, torch.float16, "output")
    info = q_matrix_info(q_handle)
    if info["height"] != output.shape[0] or info["width"] != output.shape[1]:
        raise RuntimeError("Output tensor doesn't match shape of QMatrix")
    _check(lib.exl2b_reconstruct(q_handle, output.data_ptr(), _stream(output)))


def gemm_half_q_half(a: torch.Tensor, b: int, c: torch.Tensor, force_cuda: bool = False):
    """ext_qmatrix.cpp:213-247: c = a @ W (+ bias), a fp16[M,K], c fp16[M,N]."""
    _cuda(a, "a")
    _dtype(a, torch.float16, "a")
    _dtype(c, torch.float16, "c")
    if a.shape[0] != c.shape[0]:
        raise RuntimeError("a and c have incompatible shapes")
    info = q_matrix_info(b)
    if info["height"] != a.shape[1]:
        raise RuntimeError("a and b have incompatible shapes")
    if info["width"] != c.shape[1]:
        raise RuntimeError("b and c have incompatible shapes")
    if a.stride(1) != 1 or c.stride(1) != 1:
        raise RuntimeError("a and c must be row-major")
    _check(lib.exl2b_gemm_half_q_half(b, a.data_ptr(), a.stride(0), c.data_ptr(), c.stride(0), a.shape[0], 1,
                                      int(force_cuda), _stream(a)))


def gemv_norm(x: torch.Tensor, b: int, w: torch.Tensor, epsilon: float, c: torch.Tensor, clear: bool = True, prepared: bool = False):
    """rms_norm(x, w) followed by gemm_half_q_half, fused into one launch for a single row (decode: final norm + lm_head);
    more rows run the two reference ops (rmsnorm.py:141, linear.py:366)."""
    _cuda(x, "x")
    _dtype(x, torch.float16, "x")
    _dtype(c, torch.float16, "c")
    rows = x.numel() // x.shape[-1]
    if rows == 1:
        # prepared: the row was left in the matrix's stored-row order by a chained producer launch (exl2b_chain_t)
        _check(lib.exl2b_gemm_half_q_half_norm(b, None if prepared else x.data_ptr(), w.data_ptr(), float(epsilon), c.data_ptr(),
                                               int(clear), _stream(x)))
        return
    y = torch.empty_like(x)
    rms_norm(x, w, y, epsilon)
    if clear:
        gemm_half_q_half(y.view(rows, -1), b, c.view(rows, -1), False)
    else:
        gemm_half_q_half_accum(y.view(rows, -1), b, c.view(rows, -1))


def gemm_half_q_half_accum(a: torch.Tensor, b: int, c: torch.Tensor):
    """c += a @ W -- the clear=false form the reference uses internally for residual adds (cuda/q_attn.cu:333)."""
    _check(lib.exl2b_gemm_half_q_half(b, a.data_ptr(), a.stride(0), c.data_ptr(), c.stride(0), a.shape[0], 0, 0, _stream(a)))


def gemm_half_q_half_host(a_host: torch.Tensor, b: int, c_host: torch.Tensor, device: torch.device):
    """Host-buffer entry point (bench.py e2e): copies a to the device, multiplies, copies c back, waits."""
    _check(lib.exl2b_gemm_half_q_half_host(b, a_host.data_ptr(), c_host.data_ptr(), a_host.shape[0],
                                           torch.cuda.current_stream(device).cuda_stream))


def make_group_map(q_groups: torch.Tensor, num_qrows: int) -> torch.Tensor:
    """ext_qmatrix.cpp:341-361 (CPU tensor in, CPU int16 tensor out)."""
    _dtype(q_groups, torch.int16, "q_groups")
    g = q_groups.cpu().contiguous()
    ng = g.shape[0] // 2
    bits = g[0::2].to(torch.int64)
    cap = int((num_qrows * 32 // max(1, int(bits.min()))) * 2 + 64)
    out = torch.empty((cap,), dtype=torch.int16)
    k = c_int()
    _check(lib.exl2b_make_group_map(ctypes.cast(g.data_ptr(), POINTER(c_int16)), ng, num_qrows,
                                    ctypes.cast(out.data_ptr(), POINTER(c_int16)), cap, ctypes.byref(k)))
    return out[: 2 * k.value].clone()


# ---------------------------------------------------------------------------------------------------------------
# norm / rope / activation
# ---------------------------------------------------------------------------------------------------------------

def rms_norm(x: torch.Tensor, w: torch.Tensor, y: torch.Tensor, epsilon: float):
    """ext_norm.cpp:23-62 (fp16 in / fp16 out form)."""
    _cuda(x, "x")
    _dtype(x, torch.float16, "x")
    _dtype(w, torch.float16, "w")
    _dtype(y, torch.float16, "y")
    dim = x.shape[-1]
    if w.shape[0] != dim:
        raise RuntimeError("x and w have incompatible shapes")
    rows = x.numel() // dim
    _check(lib.exl2b_rms_norm(x.data_ptr(), w.data_ptr(), y.data_ptr(), float(epsilon), rows, dim, _stream(x)))


def rms_norm_(x: torch.Tensor, w: torch.Tensor, epsilon: float):
    """ext_norm.cpp:64-103: in place."""
    rms_norm(x, w, x, epsilon)


def rope_(x: torch.Tensor, sin: torch.Tensor, cos: torch.Tensor, past_len: int, num_heads: int, head_dim: int,
          offsets: torch.Tensor, neox_style: bool):
    """ext_rope.cpp:20-62: x fp16[batch, seq, heads*head_dim] rotated in place."""
    _cuda(x, "x")
    _dtype(x, torch.float16, "x")
    _dtype(sin, torch.float16, "sin")
    _dtype(cos, torch.float16, "cos")
    if head_dim * num_heads != x.shape[-1]:
        raise RuntimeError("x has wrong last dimension for num_heads * head_dim")
    batch = x.shape[0]
    rows_per_batch = x.numel() // head_dim // batch
    sincos_size = sin.shape[-1]
    _check(lib.exl2b_rope(x.data_ptr(), sin.data_ptr(), cos.data_ptr(), batch, rows_per_batch, head_dim, num_heads,
                          int(past_len), _p(offsets), int(bool(neox_style)), sincos_size, _stream(x)))


def act_mul(x: torch.Tensor, y: torch.Tensor, act_gelu: bool = False):
    _check(lib.exl2b_act_mul(x.data_ptr(), y.data_ptr(), x.numel() // x.shape[-1], x.shape[-1], int(act_gelu), _stream(x)))


# ---------------------------------------------------------------------------------------------------------------
# Q4 / Q6 / Q8 K/V cache
# ---------------------------------------------------------------------------------------------------------------

# values per stored byte of the keys / values for each cache format (cache.py:584-656): Q4 2/2, Q6 1/2, Q8 1/1
KV_WEIGHTS_PER_BYTE = {4: (2, 2), 6: (1, 2), 8: (1, 1)}


def _check_kv_shapes(fp16_k, q_k, fp16_v, q_v, wbits):
    """The kernel derives every offset from the fp16 tensor's shape: a quantised state tensor of the wrong width for `wbits`
    would be read or written out of bounds.  (An unknown wbits is left to the library, whose error names the accepted ones.)"""
    if wbits not in KV_WEIGHTS_PER_BYTE:
        return
    for name, f, q, wpe in (("key", fp16_k, q_k, KV_WEIGHTS_PER_BYTE[wbits][0]), ("value", fp16_v, q_v, KV_WEIGHTS_PER_BYTE[wbits][1])):
        if f is None or f.is_meta or q is None or q.is_meta:
            continue
        if q.shape[-1] * wpe != f.shape[-1]:
            raise RuntimeError(f"{name} states have last dimension {q.shape[-1]}, but a wbits={wbits} cache stores "
                               f"{f.shape[-1] // wpe} bytes per {f.shape[-1]}-value row")

def _check_kv_range(fp16_k, batch_size: int, offset: int, width: int, page_size: int):
    """Non-paged: tokens [offset, offset + width) of `batch_size` rows must lie inside the fp16 tensor; the kernels then widen
    the range to whole 512-value blocks within each row and never past its end (kvcache.cu kv_common)."""
    if page_size:
        return
    if batch_size > fp16_k.shape[0] or offset < 0 or width < 0 or offset + width > fp16_k.shape[1]:
        raise RuntimeError(f"tokens [{offset}, {offset + width}) of {batch_size} rows are outside the tensor's "
                           f"{fp16_k.shape[0]} rows of {fp16_k.shape[1]} tokens")


def _kv_call(fn, a_k, b_k, s_k, a_v, b_v, s_v, fp16_k, batch_size, offset, width, page_size, cache_seqlens, block_table, wbits):
    _check_kv_range(fp16_k, batch_size, offset, width, page_size)
    dim = fp16_k.shape[2] * fp16_k.shape[3]
    seq_stride = fp16_k.shape[1] * dim
    pages = 0
    if page_size:
        batch_size = block_table.shape[0]
        pages = block_table.shape[1]
        if cache_seqlens.shape[0] != block_table.shape[0]:
            raise RuntimeError("cache_seqlens and block_table have incompatible shapes")
    _check(fn(a_k.data_ptr(), b_k.data_ptr(), s_k.data_ptr(), _p(a_v), _p(b_v), _p(s_v), batch_size, dim, seq_stride,
              offset, width, page_size, _p(cache_seqlens), _p(block_table), pages, wbits, _stream(a_k)))


def fp16_to_q_kv(k_in, k_out, k_scales, v_in, v_out, v_scales, batch_size: int, offset: int, width: int, page_size: int,
                 cache_seqlens, block_table, wbits: int):
    """ext_cache.cpp:80-174"""
    _cuda(k_in, "k_in")
    _dtype(k_in, torch.float16, "k_in")
    _dtype(k_out, torch.uint8, "k_out")
    _check_kv_shapes(k_in, k_out, v_in, v_out, wbits)
    _kv_call(lib.exl2b_fp16_to_q_kv, k_in, k_out, k_scales, v_in, v_out, v_scales, k_in, batch_size, offset, width,
             page_size, cache_seqlens, block_table, wbits)


def q_to_fp16_kv(k_in, k_out, k_scales, v_in, v_out, v_scales, batch_size: int, offset: int, width: int, page_size: int,
                 cache_seqlens, block_table, wbits: int):
    """ext_cache.cpp:176-274 (argument order of the reference: in, OUT, scales)."""
    _cuda(k_in, "k_in")
    _dtype(k_in, torch.uint8, "k_in")
    _dtype(k_out, torch.float16, "k_out")
    _check_kv_shapes(k_out, k_in, v_out, v_in, wbits)
    _check_kv_range(k_out, batch_size, offset, width, page_size)
    # C ABI order is (in, scales, out)
    dim = k_out.shape[2] * k_out.shape[3]
    seq_stride = k_out.shape[1] * dim
    pages = 0
    if page_size:
        batch_size = block_table.shape[0]
        pages = block_table.shape[1]
    _check(lib.exl2b_q_to_fp16_kv(k_in.data_ptr(), k_scales.data_ptr(), k_out.data_ptr(), _p(v_in), _p(v_scales), _p(v_out),
                                  batch_size, dim, seq_stride, offset, width, page_size, _p(cache_seqlens), _p(block_table),
                                  pages, wbits, _stream(k_in)))


# ---------------------------------------------------------------------------------------------------------------
# fused blocks
# ---------------------------------------------------------------------------------------------------------------

def make_q_attn(layernorm, layernorm_bias, layernorm_is_rms: bool, headnorm_is_rms: bool, norm_epsilon: float,
                q_q_proj: int, q_k_proj: int, q_v_proj: int, q_o_proj: int, temp_state, temp_dq, max_rows: int,
                hidden_size: int, num_heads: int, num_kv_heads: int, head_dim: int, max_seq_len: int, has_residual: bool,
                rope_style: int, sincos_size: int, q_norm, k_norm, post_layernorm, post_layernorm_bias,
                residual_fp32: bool, use_graphs: bool) -> int:
    """ext_qattn.cpp:24-104, same 26 arguments.  Llama-family subset: RMSNorm pre-norm, no QK-norm, no
    post-norm, fp16 residual stream; anything else raises (out of scope, SURVEY.md 2.2)."""
    if not layernorm.is_meta and not layernorm_is_rms:
        raise RuntimeError("exllamav2_b200: only RMSNorm pre-normalisation is implemented")
    for t, name in ((q_norm, "q_norm"), (k_norm, "k_norm"), (post_layernorm, "post_layernorm")):
        if t is not None and not t.is_meta:
            raise RuntimeError(f"exllamav2_b200: {name} is not implemented (out of scope)")
    if residual_fp32:
        raise RuntimeError("exllamav2_b200: fp32 residual stream is not implemented")
    d = _QAttnDesc()
    d.layernorm = _p(layernorm)
    d.norm_epsilon = float(norm_epsilon)
    d.q_proj, d.k_proj, d.v_proj, d.o_proj = q_q_proj, q_k_proj, q_v_proj, q_o_proj
    d.hidden_size, d.num_heads, d.num_kv_heads, d.head_dim = hidden_size, num_heads, num_kv_heads, head_dim
    d.has_residual = int(has_residual)
    d.rope_style = int(rope_style)
    d.sincos_size = int(sincos_size)
    out = c_void_p()
    _check(lib.exl2b_qattn_create(ctypes.byref(d), ctypes.byref(out)))
    return out.value


def free_q_attn(handle: int):
    _lora_keep.pop(handle, None)
    _check(lib.exl2b_qattn_destroy(handle))


def q_attn_forward_1(q_attn: int, x, batch_size: int, q_len: int, past_len: int, past_lens, q_temp, k_temp, v_temp, sin, cos,
                     loras=(), loras_temp=none_tensor):
    """ext_qattn.cpp:115-159.  loras: ids of the active adapters (id(lora), as attn.py:528-548 passes them); loras_temp is
    accepted and unused (the LoRA launch keeps x·A on chip)."""
    _cuda(x, "x")
    _dtype(x, torch.float16, "x")
    _check(lib.exl2b_qattn_forward_1(q_attn, x.data_ptr(), batch_size, q_len, int(past_len), _p(past_lens), q_temp.data_ptr(),
                                     k_temp.data_ptr(), v_temp.data_ptr(), _p(sin), _p(cos), 0, *_lora_ids(loras), _stream(x)))


def q_attn_forward_2(q_attn: int, x, attn_output, batch_size: int, q_len: int, loras=(), loras_temp=none_tensor):
    """ext_qattn.cpp:161-191 (loras / loras_temp as q_attn_forward_1)"""
    _check(lib.exl2b_qattn_forward_2(q_attn, x.data_ptr(), attn_output.data_ptr(), batch_size, q_len, 0, None, *_lora_ids(loras),
                                     _stream(x)))


# ---- LoRA (ext_qattn.cpp:194-240, ext_qmlp.cpp q_mlp_set_loras; include/exl2_b200.h "LoRA adapters on the blocks") ----------------

LORA_MAX_RANK = 512          # EXL2B_LORA_MAX_RANK: ranks (each rounded up to 8) of all adapters on one stage
LORA_MAX_ADAPTERS = 8        # EXL2B_LORA_MAX_ADAPTERS
_lora_keep: dict[int, list] = {}      # handle -> the adapter tensors it points to (kept alive while the set is registered)


def _lora_ids(loras):
    """(ids, num_ids) of the block forwards: the active adapter ids as a C array, or (NULL, 0) for none."""
    ids = [int(i) for i in loras or ()]
    return ((c_uint64 * len(ids))(*ids) if ids else None), len(ids)


def _lora_set(projs) -> tuple:
    """projs: [(name, a_dict, b_dict)] in the block's projection order, dicts keyed by adapter id (id(lora), attn.py:1545-1552).
    Checks every tensor (shape checks against the matrices are the library's) and returns the C array and its length."""
    ids = []
    for _, a, b in projs:
        for key in list(a) + list(b):
            if key not in ids:
                ids.append(key)
    if len(ids) > LORA_MAX_ADAPTERS:
        raise RuntimeError(f"LoRA: {len(ids)} adapters given, a block holds at most {LORA_MAX_ADAPTERS}")
    arr = (_Lora * max(1, len(ids)))()
    for i, key in enumerate(ids):
        arr[i].id = int(key)
        for p, (name, a_dict, b_dict) in enumerate(projs):
            a, b = a_dict.get(key), b_dict.get(key)
            if a is None and b is None:
                continue
            if a is None or b is None:
                raise RuntimeError(f"LoRA adapter {key}: {name} has {'A' if b is None else 'B'} but no {'B' if b is None else 'A'}")
            for t, what in ((a, f"{name} lora_a"), (b, f"{name} lora_b")):
                if t.dim() != 2:
                    raise RuntimeError(f"LoRA adapter {key}: {what} must be 2-D, got shape {tuple(t.shape)}")
                _dtype(t, torch.float16, what)
                if not t.is_contiguous():
                    raise RuntimeError(f"LoRA adapter {key}: {what} must be contiguous")
            r = a.shape[1]
            if b.shape[0] != r:
                raise RuntimeError(f"LoRA adapter {key}: {name} A {tuple(a.shape)} and B {tuple(b.shape)} have incompatible shapes")
            if not 1 <= (r + 7) // 8 * 8 <= LORA_MAX_RANK:
                raise RuntimeError(f"LoRA adapter {key}: {name} rank {r} is outside 1..{LORA_MAX_RANK} (LORA_MAX_RANK)")
            _cuda(a, f"{name} lora_a")
            _cuda(b, f"{name} lora_b")
            arr[i].a[p], arr[i].b[p] = a.data_ptr(), b.data_ptr()
            arr[i].rank[p], arr[i].a_rows[p], arr[i].b_cols[p] = r, a.shape[0], b.shape[1]
    return arr, len(ids)


def _set_loras(fn, handle: int, projs) -> int:
    arr, n = _lora_set(projs)
    mr = c_int(0)
    _check(fn(handle, arr, n, ctypes.byref(mr)))
    _lora_keep[handle] = [t for _, a, b in projs for d in (a, b) for t in d.values()]
    return mr.value


def q_attn_set_loras(q_attn: int, q_proj_lora_a: dict, q_proj_lora_b: dict, k_proj_lora_a: dict, k_proj_lora_b: dict,
                     v_proj_lora_a: dict, v_proj_lora_b: dict, o_proj_lora_a: dict, o_proj_lora_b: dict) -> int:
    """ext_qattn.cpp:194-240: replace the handle's adapters; returns the largest rank (attn.py:1554 sizes temp_lora with it)."""
    return _set_loras(lib.exl2b_qattn_set_loras, q_attn, [("q_proj", q_proj_lora_a, q_proj_lora_b), ("k_proj", k_proj_lora_a, k_proj_lora_b),
                                                          ("v_proj", v_proj_lora_a, v_proj_lora_b), ("o_proj", o_proj_lora_a, o_proj_lora_b)])


def q_mlp_set_loras(q_mlp: int, gate_proj_lora_a: dict, gate_proj_lora_b: dict, up_proj_lora_a: dict, up_proj_lora_b: dict,
                    down_proj_lora_a: dict, down_proj_lora_b: dict) -> int:
    """ext_qmlp.cpp q_mlp_set_loras (called from mlp.py:536): as q_attn_set_loras."""
    return _set_loras(lib.exl2b_qmlp_set_loras, q_mlp, [("gate_proj", gate_proj_lora_a, gate_proj_lora_b),
                                                        ("up_proj", up_proj_lora_a, up_proj_lora_b),
                                                        ("down_proj", down_proj_lora_a, down_proj_lora_b)])


def lora_stack(ranks) -> tuple[list, int]:
    """How one launch stacks adapters (host only, include/exl2_b200.h exl2b_lora_stack): ranks [adapters][projections] (0: none)
    -> ([(adapter, projection, first stacked column)], stacked width).  Raises past LORA_MAX_RANK."""
    na, npj = len(ranks), len(ranks[0])
    flat = (c_int * (na * npj))(*[int(r) for row in ranks for r in row])
    sa, sp, so = (c_int * 32)(), (c_int * 32)(), (c_int * 32)()
    ns, tot = c_int(), c_int()
    _check(lib.exl2b_lora_stack(flat, na, npj, sa, sp, so, ctypes.byref(ns), ctypes.byref(tot)))
    return [(sa[i], sp[i], so[i]) for i in range(ns.value)], tot.value


def make_q_mlp(layernorm, layernorm_bias, layernorm_is_rms: bool, norm_epsilon: float, q_gate: int, q_up: int, q_down: int,
               temp_state, temp_a, temp_b, temp_dq, max_rows: int, act_gelu: bool, has_residual: bool, post_layernorm,
               post_layernorm_bias, residual_fp32: bool, use_graphs: bool) -> int:
    """ext_qmlp.cpp:22-85, same arguments.  temp_a / temp_b are remembered per handle like the reference does."""
    if not layernorm.is_meta and not layernorm_is_rms:
        raise RuntimeError("exllamav2_b200: only RMSNorm pre-normalisation is implemented")
    if post_layernorm is not None and not post_layernorm.is_meta:
        raise RuntimeError("exllamav2_b200: post_layernorm is not implemented (out of scope)")
    if residual_fp32:
        raise RuntimeError("exllamav2_b200: fp32 residual stream is not implemented")
    if not q_gate:
        raise RuntimeError("exllamav2_b200: un-gated MLP is not implemented (out of scope)")
    gi, ui = q_matrix_info(q_gate), q_matrix_info(q_up)
    d = _QMlpDesc()
    d.layernorm = _p(layernorm)
    d.norm_epsilon = float(norm_epsilon)
    d.gate, d.up, d.down = q_gate, q_up, q_down
    d.hidden_size = gi["height"]
    d.intermediate_size = ui["width"]
    d.act_gelu = int(act_gelu)
    d.has_residual = int(has_residual)
    out = c_void_p()
    _check(lib.exl2b_qmlp_create(ctypes.byref(d), ctypes.byref(out)))
    _mlp_temps[out.value] = (temp_a, temp_b)
    _mlp_dims[out.value] = (d.hidden_size, d.intermediate_size)
    return out.value


_mlp_temps: dict[int, tuple] = {}
_mlp_dims: dict[int, tuple] = {}      # handle -> (hidden size, intermediate size): row widths of x and of act(gate) * up


def q_mlp_forward_rows(q_mlp: int, x, temp_a, temp_b, loras=(), loras_temp=none_tensor):
    """q_mlp_forward_ with caller-provided scratch rows (the reference sizes temp_a / temp_b for max_input_len at make_q_mlp
    time, mlp.py:176-203; a prompt chunk larger than that brings its own)."""
    _cuda(x, "x")
    _dtype(x, torch.float16, "x")
    rows = x.numel() // x.shape[-1]
    _check(lib.exl2b_qmlp_forward(q_mlp, x.data_ptr(), rows, temp_a.data_ptr(), temp_b.data_ptr(), 0, None, *_lora_ids(loras),
                                  _stream(x)))


def free_q_mlp(handle: int):
    _mlp_temps.pop(handle, None)
    _mlp_dims.pop(handle, None)
    _lora_keep.pop(handle, None)
    _check(lib.exl2b_qmlp_destroy(handle))


def q_mlp_forward_(q_mlp: int, x, loras=(), loras_temp=none_tensor):
    """ext_qmlp.cpp:87-118: x is updated in place (loras / loras_temp as q_attn_forward_1)."""
    _cuda(x, "x")
    _dtype(x, torch.float16, "x")
    temp_a, temp_b = _mlp_temps[q_mlp]
    rows = x.numel() // x.shape[-1]
    if rows > temp_a.shape[0]:          # the reference sizes temp_a / temp_b for max_rows at make_q_mlp time and would write past them
        raise RuntimeError(f"q_mlp_forward_: {rows} rows exceed the {temp_a.shape[0]} rows of temp_a given to make_q_mlp "
                           "(use q_mlp_forward_rows with scratch of your own for larger chunks)")
    _check(lib.exl2b_qmlp_forward(q_mlp, x.data_ptr(), rows, temp_a.data_ptr(), _p(temp_b), 0, None, *_lora_ids(loras), _stream(x)))


# names the reference's hot-path call sites use (SURVEY.md 8b) that this module provides

def q_mlp_forward_gateup(q_mlp: int, x, temp_a):
    """temp_a[rows, intermediate] = act(norm(x) @ gate) * (norm(x) @ up) -- the first half of q_mlp_forward_, used by a
    tensor-parallel rank on its intermediate slice (ext_qmlp.cpp:326-473).  The launch reads rows x hidden values from x's first
    element on and writes rows x intermediate values from temp_a's, so both must be contiguous rows of those widths and temp_a
    must hold the rows: checked here, before anything is launched."""
    for t, what in ((x, "x"), (temp_a, "temp_a")):
        _cuda(t, what)
        _dtype(t, torch.float16, what)
        if not t.is_contiguous():
            raise RuntimeError(f"q_mlp_forward_gateup: {what} must be contiguous, got shape {tuple(t.shape)} strides {t.stride()}")
    hidden, inter = _mlp_dims[q_mlp]
    if x.shape[-1] != hidden:
        raise RuntimeError(f"q_mlp_forward_gateup: x rows are {x.shape[-1]} wide, the handle's hidden size is {hidden}")
    rows = x.numel() // hidden
    if temp_a.dim() != 2 or temp_a.shape[1] != inter:
        raise RuntimeError(f"q_mlp_forward_gateup: temp_a must be [rows, {inter}] (the handle's intermediate size), "
                           f"got shape {tuple(temp_a.shape)}")
    if temp_a.shape[0] < rows:
        raise RuntimeError(f"q_mlp_forward_gateup: {rows} rows of x exceed the {temp_a.shape[0]} rows of temp_a")
    _check(lib.exl2b_qmlp_forward_gateup(q_mlp, x.data_ptr(), rows, temp_a.data_ptr(), _stream(x)))


def make_chain(consumers, norm_weight=None) -> "_Chain":
    """Describe who reads a launch's output: `consumers` = q_handles of the matrices fed by it, `norm_weight` = the
    RMSNorm weight they apply (include/exl2_b200.h exl2b_chain_t).  Keep the returned object (and norm_weight) alive."""
    c = _Chain()
    for i, hnd in enumerate(consumers):
        c.consumers[i] = hnd
    c.num_consumers = len(consumers)
    c.norm_weight = _p(norm_weight)
    c._keep = norm_weight
    return c


def q_attn_forward_1_ex(q_attn: int, x, batch_size: int, q_len: int, past_len: int, past_lens, q_temp, k_temp, v_temp, sin, cos,
                        input_prepared: bool, loras=()):
    """loras: active adapter ids (as q_attn_forward_1); a chained call with adapters takes one row (include/exl2_b200.h
    "block forwards")"""
    _check(lib.exl2b_qattn_forward_1(q_attn, _p(x), batch_size, q_len, int(past_len), _p(past_lens), q_temp.data_ptr(),
                                     k_temp.data_ptr(), v_temp.data_ptr(), _p(sin), _p(cos), int(input_prepared), *_lora_ids(loras),
                                     _stream(q_temp)))


def q_attn_forward_2_ex(q_attn: int, x, attn_output, batch_size: int, q_len: int, input_prepared: bool, chain=None, loras=()):
    ch = ctypes.byref(chain) if chain is not None else None
    _check(lib.exl2b_qattn_forward_2(q_attn, x.data_ptr(), _p(attn_output), batch_size, q_len, int(input_prepared), ch,
                                     *_lora_ids(loras), _stream(x)))


def q_mlp_forward_ex(q_mlp: int, x, input_prepared: bool, chain=None, loras=()):
    temp_a, temp_b = _mlp_temps[q_mlp]
    rows = x.numel() // x.shape[-1]
    ch = ctypes.byref(chain) if chain is not None else None
    _check(lib.exl2b_qmlp_forward(q_mlp, x.data_ptr(), rows, temp_a.data_ptr(), _p(temp_b), int(input_prepared), ch,
                                  *_lora_ids(loras), _stream(x)))


def gemm_half_q_half_prepared(b: int, c, has_norm: bool, norm_eps: float, clear: bool = True):
    _check(lib.exl2b_gemm_half_q_half_prepared(b, c.data_ptr(), c.stride(0), c.shape[0], int(clear), int(has_norm),
                                               float(norm_eps), _stream(c)))


def paged_attn_decode_q4(q, k_new, v_new, k_cache, k_scales, v_cache, v_scales, cache_seqlens, block_table, out,
                         softmax_scale: float, out_consumer: int = 0, rope=None, wbits: int = 4):
    """Decode attention over the paged Q4 / Q6 / Q8 cache (`wbits` as fp16_to_q_kv) with quantise-and-append of the new rows
    (include/exl2_b200.h exl2b_paged_attn_decode_q).  q [B, q_len, H, hd]; k_new / v_new [B, q_len, KVH, hd]; caches uint8
    [pages, page, KVH, hd/2] (4-bit) or [pages, page, KVH, hd] (8-bit) + fp16 scales [pages, page, KVH, hd/32]; out like q.
    No reference counterpart as one op: it replaces q_to_fp16_kv + flash_attn_with_kvcache + fp16_to_q_kv (attn.py:560-613)."""
    B, q_len, H, hd = q.shape
    KVH = k_new.shape[2]
    for t in (q, k_new, v_new, out):
        _dtype(_cuda(t, "attention operand"), torch.half, "attention operand")
    _check_kv_shapes(k_new, k_cache, v_new, v_cache, wbits)
    # rope = (sin, cos, rope_style): q / k_new are the un-rotated projection outputs, rotated as the kernel reads them
    sin, cos, style = rope if rope is not None else (None, None, 0)
    _check(lib.exl2b_paged_attn_decode_q(
        _p(q), _p(k_new), _p(v_new), _p(k_cache), _p(k_scales), _p(v_cache), _p(v_scales),
        _p(cache_seqlens), _p(block_table), _p(out), B, q_len, H, KVH, hd, k_cache.shape[1], block_table.shape[1],
        float(softmax_scale), out_consumer or None, _p(sin), _p(cos), int(style), sin.shape[-1] if sin is not None else 0,
        int(wbits), _stream(q)))


def paged_attn_prefill_q(q, k_new, v_new, k_cache, k_scales, v_cache, v_scales, cache_seqlens, block_table, out,
                         softmax_scale: float, wbits: int = 4):
    """Prompt attention over the paged Q4 / Q6 / Q8 cache for any q_len, with quantise-and-append of the new rows (include/
    exl2_b200.h exl2b_paged_attn_prefill_q).  Shapes as paged_attn_decode_q4; q is RoPE-rotated already.  No reference
    counterpart as one op: it replaces q_to_fp16_kv + flash_attn_with_kvcache + fp16_to_q_kv (attn.py:560-621)."""
    B, q_len, H, hd = q.shape
    KVH = k_new.shape[2]
    for t in (q, k_new, v_new, out):
        _dtype(_cuda(t, "attention operand"), torch.half, "attention operand")
    for t, dt, what in ((k_cache, torch.uint8, "k_cache"), (v_cache, torch.uint8, "v_cache"), (k_scales, torch.half, "k_scales"),
                        (v_scales, torch.half, "v_scales"), (cache_seqlens, torch.int32, "cache_seqlens"),
                        (block_table, torch.int32, "block_table")):
        _dtype(_cuda(t, what), dt, what)
    _check_kv_shapes(k_new, k_cache, v_new, v_cache, wbits)
    if tuple(k_new.shape) != (B, q_len, KVH, hd) or tuple(v_new.shape) != (B, q_len, KVH, hd) or tuple(out.shape) != (B, q_len, H, hd):
        raise RuntimeError(f"k_new / v_new must be [{B}, {q_len}, KVH, {hd}] and out [{B}, {q_len}, {H}, {hd}]; got "
                           f"{tuple(k_new.shape)}, {tuple(v_new.shape)}, {tuple(out.shape)}")
    if tuple(k_cache.shape[2:3]) != (KVH,) or k_scales.shape[-1] * 32 != hd or v_scales.shape[-1] * 32 != hd:
        raise RuntimeError(f"cache tensors must be [pages, page_size, {KVH}, ...] with {hd // 32} scales per row")
    if block_table.dim() != 2 or cache_seqlens.shape[0] != block_table.shape[0] or block_table.shape[0] != B:
        raise RuntimeError("cache_seqlens and block_table have incompatible shapes")
    for t in (q, k_new, v_new, out, k_cache, k_scales, v_cache, v_scales, cache_seqlens, block_table):
        if not t.is_contiguous():
            raise RuntimeError("attention operands must be contiguous")
    _check(lib.exl2b_paged_attn_prefill_q(
        _p(q), _p(k_new), _p(v_new), _p(k_cache), _p(k_scales), _p(v_cache), _p(v_scales), _p(cache_seqlens), _p(block_table),
        _p(out), B, q_len, H, KVH, hd, k_cache.shape[1], block_table.shape[1], float(softmax_scale), int(wbits), _stream(q)))


def paged_attn_clear_status(device) -> None:
    _check(lib.exl2b_paged_attn_clear_status(torch.device(device).index or 0))


def paged_attn_status(device) -> int:
    """Sticky error bits of the fused attention kernels (bit 0: a sequence ran past its page table).  Synchronises."""
    st = c_int(0)
    _check(lib.exl2b_paged_attn_status(torch.device(device).index or 0, ctypes.byref(st)))
    return st.value


# include/exl2_b200.h EXL2B_SCRATCH_*
SCRATCH_KINDS = {"attn_ws": 0, "attn_cnt": 1, "tc_ws": 2, "tc_cnt": 3, "tc_xp": 4, "tc_ws_wide": 5, "tc_xp_wide": 6}


def debug_scratch(device, stream, kind: str) -> tuple[int, int]:
    """(device address, bytes) of the scratch a kernel family keeps for (device, stream) -- `kind` one of SCRATCH_KINDS --
    or (0, 0) before the first launch that creates it.  `stream` is a torch.cuda.Stream or a raw cudaStream_t handle."""
    handle = stream.cuda_stream if hasattr(stream, "cuda_stream") else int(stream)
    ptr, nbytes = c_void_p(), ctypes.c_size_t()
    _check(lib.exl2b_debug_scratch(torch.device(device).index or 0, handle or None, SCRATCH_KINDS[kind], ctypes.byref(ptr),
                                   ctypes.byref(nbytes)))
    return ptr.value or 0, nbytes.value


HOT_PATH_EXPORTS = [
    "make_q_matrix", "free_q_matrix", "reconstruct", "gemm_half_q_half", "make_group_map",
    "rms_norm", "rms_norm_", "rope_", "fp16_to_q_kv", "q_to_fp16_kv",
    "make_q_attn", "free_q_attn", "q_attn_forward_1", "q_attn_forward_2",
    "make_q_mlp", "free_q_mlp", "q_mlp_forward_", "q_attn_set_loras", "q_mlp_set_loras",
]


# Names of the reference extension that are NOT on the hot path (sampling, safetensors loader, MoE, head / layer norm,
# FP8 cache, converter kernels, the single-process TP glue -- SURVEY.md 2.2) are forwarded to the stock extension when the
# deployment registers one; otherwise the AttributeError says exactly which name is missing and why.
_stock_ext = None


def set_stock_extension(module) -> None:
    """Register the reference's own build of `exllamav2_ext` (or any module exporting its names) as the provider of
    everything outside the hot path."""
    global _stock_ext
    _stock_ext = module


def __getattr__(name: str):
    if name.startswith("__"):
        raise AttributeError(name)
    stock = _stock_ext
    if stock is None:
        try:
            import importlib
            stock = importlib.import_module("exllamav2_ext_stock")      # a deployment may put the stock build on sys.path under this name
            set_stock_extension(stock)
        except ImportError:
            stock = None
    if stock is not None and hasattr(stock, name):
        return getattr(stock, name)
    raise AttributeError(f"exllamav2_b200.ext: '{name}' is outside the quantized-linear hot path this module replaces and no stock "
                         f"exllamav2_ext is registered (exllamav2_b200.ext.set_stock_extension / module 'exllamav2_ext_stock')")


def install_as_exllamav2_ext():
    """Register this module under the name the reference imports (exllamav2/ext.py:106-109 does
    `import exllamav2_ext` first and only JIT-builds its own extension when that fails)."""
    sys.modules["exllamav2_ext"] = sys.modules[__name__]
