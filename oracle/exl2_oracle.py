"""CPU restatement (numpy) of the reference's quantized-linear hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under exllamav2_b200/ (the product) may import this module; only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs use it, and only as the checker.

Parity status: PINNED against the reference extension itself.  The reference holds no golden vectors for this
path (SURVEY.md 8c), so `oracle/gen_golden.py` runs the unmodified reference CUDA extension (built by
oracle/build_ref.py into oracle/_ref/) on a GPU over the seeded tensors from `oracle/synth.py` and stores its
outputs under tests/golden/; tests/test_oracle_golden.py checks every function below against them.

All citations are path:line relative to exllamav2/ in the reference checkout.

Formats (SURVEY.md Appendix B):
  EXL2  q_weight int32[R,N]  bit-strips in descending bit width; within a strip each column is a little-endian
        bit stream down K (exllamav2_ext/cuda/pack_tensor.cu:118-271; decode = the non-shuffled branches of
        exllamav2_ext/cuda/quant/qdq_{2,3,4,5,6,8}.cuh)
        q_scale int32[G,N/8] nibble n%8 of word n/8, stored = qscale-1 (cuda/matrix_view.cuh:96-118,
        cuda/pack_tensor.cu:10-36); q_scale_max fp16[G]; q_groups int16[2G] = (bits, first packed row);
        q_invperm int32[K]; q_perm = argsort(q_invperm) (module.py:120)
  GPTQ  qweight int32[K/8,N] (nibble i of word r = row 8r+i), qzeros int32[G,N/8], scales fp16[G,N], g_idx
"""
from __future__ import annotations

import numpy as np

F16 = np.float16
F32 = np.float32


# --------------------------------------------------------------------------------------------------------------
# group bookkeeping
# --------------------------------------------------------------------------------------------------------------

def exl2_group_rows(q_groups: np.ndarray, num_qrows: int, height: int | None = None):
    """Rows of K covered by each group.  exllamav2_ext/cuda/q_matrix.cu:130-150 and ext.py:301-316.

    Returns (bits[G], first_qrow[G], rows[G]).  The last group runs to the end of the packed tensor."""
    g = np.asarray(q_groups).astype(np.int64).reshape(-1, 2)
    bits = g[:, 0].copy()
    first = g[:, 1].copy()
    nxt = np.concatenate([first[1:], [num_qrows]])
    rows = (nxt - first) * 32 // bits
    if height is not None:
        rows[-1] = height - rows[:-1].sum()      # q_matrix.cu:150  (rows = height - row for the last group)
    return bits, first, rows


def make_group_map(q_groups: np.ndarray, num_qrows: int) -> np.ndarray:
    """(group index, rows left in group) per k row.  exllamav2_ext/ext_qmatrix.cpp:341-361."""
    bits, first, rows = exl2_group_rows(q_groups, num_qrows)
    out = []
    for i, r in enumerate(rows):
        for j in range(int(r)):
            out += [i, int(r) - j]
    return np.asarray(out, dtype=np.int16)


# --------------------------------------------------------------------------------------------------------------
# EXL2 unpack / reconstruct
# --------------------------------------------------------------------------------------------------------------

def unpack_bitstream(words: np.ndarray, bits: int, count: int) -> np.ndarray:
    """words uint32[R, N] -> q uint8/int32[count, N]: value i of a column sits at bit i*bits of the column's
    little-endian stream (qdq_2.cuh:88-99, qdq_3.cuh:148-165, qdq_4.cuh:151-162, qdq_5.cuh:179-203,
    qdq_6.cuh:130-147, qdq_8.cuh:21-34; exb() two-word funnel shift qdq_util.cuh:44-51)."""
    w = np.ascontiguousarray(words).view(np.uint32).astype(np.uint64)
    R, N = w.shape
    idx = np.arange(count, dtype=np.int64) * bits
    wi = idx // 32
    sh = (idx % 32).astype(np.uint64)
    lo = w[wi]
    hi = w[np.minimum(wi + 1, R - 1)]
    both = lo | (hi << np.uint64(32))
    q = (both >> sh[:, None]) & np.uint64((1 << bits) - 1)
    return q.astype(np.int32)


def exl2_unpack_q(q_weight: np.ndarray, q_groups: np.ndarray, height: int) -> tuple[np.ndarray, np.ndarray]:
    """Integer weights q[K,N] (stored row order k') and the group index of every row."""
    qw = np.ascontiguousarray(q_weight).view(np.uint32)
    bits, first, rows = exl2_group_rows(q_groups, qw.shape[0], height)
    N = qw.shape[1]
    q = np.zeros((height, N), dtype=np.int32)
    grp = np.zeros((height,), dtype=np.int32)
    k = 0
    for gi, (b, f, r) in enumerate(zip(bits, first, rows)):
        b, f, r = int(b), int(f), int(r)
        nq = r * b // 32
        q[k:k + r] = unpack_bitstream(qw[f:f + nq], b, r)
        grp[k:k + r] = gi
        k += r
    assert k == height
    return q, grp


def exl2_scales(q_scale: np.ndarray, q_scale_max_pre: np.ndarray, N: int) -> np.ndarray:
    """fp16 scale per (group, column): half(int2half((s+1)^2) * max) with max already multiplied by prescale/256
    in fp16 (ext.py:336).  cuda/quant/qdq_util.cuh:24-30."""
    qs = np.ascontiguousarray(q_scale).view(np.uint32)
    G = qs.shape[0]
    n = np.arange(N)
    nib = (qs[:, n // 8] >> ((n % 8) * 4).astype(np.uint32)) & 0xF
    sq = ((nib.astype(np.int32) + 1) ** 2).astype(F16)                 # exact (<= 256)
    return (sq * np.asarray(q_scale_max_pre, dtype=F16).reshape(G, 1)).astype(F16)


def prescale_max(q_scale_max: np.ndarray, prescale: float = 1.0) -> np.ndarray:
    """w["q_scale_max"] *= prescale / 256 done on an fp16 tensor (ext.py:336): torch computes the product of the
    fp16 value with the python scalar in fp32 (opmath) and rounds once to fp16."""
    return (np.asarray(q_scale_max, dtype=F16).astype(F32) * F32(prescale / 256)).astype(F16)


def exl2_reconstruct(w: dict, prescale: float = 1.0) -> np.ndarray:
    """fp16 W[K,N] in ORIGINAL row order.  b[perm[k'], n] = half(q - 2^(b-1)) * half(scale), one fp16 rounding.
    cuda/q_matrix.cu:328-497 (reconstruct_kernel), scatter at :410."""
    qw = np.asarray(w["q_weight"])
    N = qw.shape[1]
    K = int(np.asarray(w["q_invperm"]).shape[0]) if "q_invperm" in w else None
    if K is None:
        bits, first, rows = exl2_group_rows(w["q_groups"], qw.shape[0])
        K = int(rows.sum())
    q, grp = exl2_unpack_q(qw, w["q_groups"], K)
    bits, _, _ = exl2_group_rows(w["q_groups"], qw.shape[0], K)
    zp = (1 << (bits[grp] - 1)).astype(np.int32)
    sc = exl2_scales(w["q_scale"], prescale_max(w["q_scale_max"], prescale), N)
    deq = ((q - zp[:, None]).astype(F16) * sc[grp]).astype(F16)          # single fp16 multiply
    if "q_invperm" in w:
        perm = np.argsort(np.asarray(w["q_invperm"]).astype(np.int64), kind="stable")   # module.py:120
        out = np.empty_like(deq)
        out[perm] = deq
        return out
    return deq


# --------------------------------------------------------------------------------------------------------------
# GPTQ
# --------------------------------------------------------------------------------------------------------------

def gptq_groupsize(K: int, groups: int) -> int:
    """cuda/q_matrix.cu:99-105: smallest power of two with groupsize*groups >= height."""
    gs = 1
    while gs * groups < K:
        gs *= 2
    return gs


def gptq_make_sequential(g_idx: np.ndarray, groups: int) -> tuple[np.ndarray, np.ndarray]:
    """Stable group-sorted row permutation.  cuda/q_matrix.cu:597-647.  Returns (q_perm[new]=old, q_invperm)."""
    g_idx = np.asarray(g_idx).astype(np.int64)
    K = g_idx.shape[0]
    cnt = np.bincount(g_idx, minlength=groups)
    start = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    inv = np.empty(K, dtype=np.int64)
    nxt = start.copy()
    for row in range(K):
        g = g_idx[row]
        inv[row] = nxt[g]
        nxt[g] += 1
    perm = np.empty(K, dtype=np.int64)
    perm[inv] = np.arange(K)
    return perm, inv


def gptq_has_act_order(g_idx) -> bool:
    """ext.py:371: act-order path is taken iff g_idx is present and not all zero."""
    return g_idx is not None and not bool((np.asarray(g_idx) == 0).all())


def gptq_reconstruct(w: dict, offset_qzeros: bool = False) -> np.ndarray:
    """W[k,n] = half(scales[g,n]) * half(q - (zeros[g,n] + 1)).  cuda/q_matrix.cu:204-323,
    cuda/q_gemm_kernel_gptq.cuh:167-172; gptq_v2 zeros get -0x11111111 first (ext.py:366-367)."""
    qw = np.ascontiguousarray(w["qweight"]).view(np.uint32)
    qz = np.ascontiguousarray(w["qzeros"]).view(np.uint32).copy()
    if offset_qzeros:
        qz = (qz - np.uint32(0x11111111)).astype(np.uint32)
    sc = np.asarray(w["scales"], dtype=F16)
    K = qw.shape[0] * 8
    N = qw.shape[1]
    G = qz.shape[0]
    gs = gptq_groupsize(K, G)
    q = unpack_bitstream(qw, 4, K)                                          # rows in file order
    n = np.arange(N)
    z = ((qz[:, n // 8] >> ((n % 8) * 4).astype(np.uint32)) & 0xF).astype(np.int32)
    g_idx = w.get("g_idx")
    if gptq_has_act_order(g_idx):
        perm, inv = gptq_make_sequential(g_idx, G)
        qs = q[perm]                                                        # stored row k' = old row perm[k']
        grp = np.arange(K) // gs
        deq = (sc[grp] * (qs - (z[grp] + 1)).astype(F16)).astype(F16)
        out = np.empty_like(deq)
        out[perm] = deq
        return out
    grp = np.arange(K) // gs
    return (sc[grp] * (q - (z[grp] + 1)).astype(F16)).astype(F16)


# --------------------------------------------------------------------------------------------------------------
# GEMM truth: the reference is not bit-reproducible (fp16 atomics, q_gemm_kernel.cuh:560-561), so the oracle for
# gemm_half_q_half is y = a @ W_fp16 accumulated in fp64 and rounded once to fp16 (SURVEY.md 8c tolerance row).
# --------------------------------------------------------------------------------------------------------------

def gemm_truth(a: np.ndarray, W: np.ndarray, bias: np.ndarray | None = None, c_in: np.ndarray | None = None):
    y = np.asarray(a, dtype=F16).astype(np.float64) @ np.asarray(W, dtype=F16).astype(np.float64)
    if bias is not None:
        y = y + np.asarray(bias, dtype=F16).astype(np.float64)
    if c_in is not None:
        y = y + np.asarray(c_in, dtype=F16).astype(np.float64)
    return y


def rel_l2(x, ref) -> float:
    x = np.asarray(x, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    d = np.linalg.norm(ref)
    return float(np.linalg.norm(x - ref) / (d if d > 0 else 1.0))


# --------------------------------------------------------------------------------------------------------------
# RMSNorm / RoPE / activation
# --------------------------------------------------------------------------------------------------------------

def rms_norm(x: np.ndarray, w: np.ndarray, eps: float) -> np.ndarray:
    """cuda/rms_norm.cu:55-143: clamp to +-65504, sum of squares in fp32, rsqrt(mean+eps), y = half_rn(x*w*r)
    with the two products in fp32.  (Summation order differs from the CUDA tree -> <=1 fp16 ulp vs the GPU.)"""
    xf = np.clip(np.asarray(x, dtype=F16).astype(F32), -65504.0, 65504.0)
    dim = xf.shape[-1]
    s = (xf.astype(np.float64) ** 2).sum(-1, keepdims=True)
    r = (1.0 / np.sqrt(s * (1.0 / dim) + eps)).astype(F32)
    wf = np.asarray(w, dtype=F16).astype(F32)
    return ((xf * wf).astype(F32) * r).astype(F16)


def rope_tables(head_dim: int, max_seq_len: int, base: float = 10000.0, scale: float = 1.0):
    """device.py:118-170 (default rope): inv_freq = 1/base^(2i/d); t = arange/scale; freqs outer; emb = cat(f,f);
    sin/cos computed in fp32 then .half()."""
    inv_freq = 1.0 / (base ** (np.arange(0, head_dim, 2, dtype=F32) / F32(head_dim)))
    t = np.arange(max_seq_len, dtype=F32) / F32(scale)
    freqs = np.outer(t, inv_freq).astype(F32)
    emb = np.concatenate([freqs, freqs], axis=-1)
    return np.sin(emb).astype(F16), np.cos(emb).astype(F16)


def rope_neox(x: np.ndarray, sin: np.ndarray, cos: np.ndarray, pos: np.ndarray, rot: int | None = None) -> np.ndarray:
    """x [tokens, heads, head_dim] fp16, pos[tokens].  cuda/rope.cu:52-67: only the first half of the table is
    read; l' = fma(l, cos, half(r * -sin)); r' = fma(r, cos, half(l * sin)); every op rounds to fp16.
    rot: rotary width (the table's sincos_size, default head_dim); dimensions rot.. pass through unchanged."""
    x = np.asarray(x, dtype=F16)
    rot = x.shape[-1] if rot is None else rot
    h = rot // 2
    c = cos[pos, :h][:, None, :].astype(F32)
    s = sin[pos, :h][:, None, :].astype(F32)
    l = x[..., :h].astype(F32)
    r = x[..., h:rot].astype(F32)
    ls = (r * (-s)).astype(F16).astype(F32)
    rs = (l * s).astype(F16).astype(F32)
    lo = (l.astype(np.float64) * c + ls).astype(F16)      # fma: exact product + addend, one rounding
    ro = (r.astype(np.float64) * c + rs).astype(F16)
    return np.concatenate([lo, ro, x[..., rot:]], axis=-1)


def rope_gptj(x: np.ndarray, sin: np.ndarray, cos: np.ndarray, pos: np.ndarray, rot: int | None = None) -> np.ndarray:
    """cuda/rope.cu:111-122: interleaved pairs, r = fma(x_swapped, (-sin_i, +sin_{i+1}), half(x * cos)).
    rot: rotary width as in rope_neox."""
    x = np.asarray(x, dtype=F16)
    rot = x.shape[-1] if rot is None else rot
    xr = x[..., :rot]
    c = cos[pos, :rot][:, None, :].astype(F32)
    s = sin[pos, :rot][:, None, :].astype(F32).copy()
    s[..., 0::2] = -s[..., 0::2]
    xs = np.empty_like(xr)
    xs[..., 0::2] = xr[..., 1::2]
    xs[..., 1::2] = xr[..., 0::2]
    r = (xr.astype(F32) * c).astype(F16).astype(np.float64)
    return np.concatenate([(xs.astype(np.float64) * s + r).astype(F16), x[..., rot:]], axis=-1)


def silu_mul(gate: np.ndarray, up: np.ndarray) -> np.ndarray:
    """cuda/q_mlp_activation.cuh:13-35: x * hrcp(1 + hexp(-x)) in fp16, then * up in fp16.  hexp/hrcp are
    approximate intrinsics, so the oracle is exact-math rounded per step (few-ulp tolerance vs the GPU)."""
    g = np.asarray(gate, dtype=F16)
    e = np.exp(-g.astype(np.float64)).astype(F16)
    sm = (F16(1.0) + e).astype(F16)
    with np.errstate(divide="ignore", over="ignore"):
        r = (1.0 / sm.astype(np.float64)).astype(F16)
    a = (g * r).astype(F16)
    return (a * np.asarray(up, dtype=F16)).astype(F16)


def gelu_mul(gate: np.ndarray, up: np.ndarray) -> np.ndarray:
    """cuda/q_mlp_activation.cuh:24-35, line by line: t = c * (x + 0.044715 x^3) in fp32 (left to right), then
    0.5f * x * (1.0 + tanh(t)) -- the 1.0 is a double, so the last product is formed in double and narrowed to the fp32
    variable before __float2half_rn; then * up in fp16.  tanh is exact here (the GPU uses an approximation: few-ulp
    tolerance, as for silu_mul)."""
    x = np.asarray(gate, dtype=F16).astype(F32)
    t = (F32(0.797884560803) * (x + ((F32(0.044715) * x) * x) * x)).astype(F32)
    th = np.tanh(t.astype(np.float64)).astype(F32)
    h = (F32(0.5) * x).astype(F32).astype(np.float64) * (1.0 + th.astype(np.float64))
    a = h.astype(F32).astype(F16)
    return (a * np.asarray(up, dtype=F16)).astype(F16)


# --------------------------------------------------------------------------------------------------------------
# Q4 KV cache  (cuda/cache_q.cuh)
# --------------------------------------------------------------------------------------------------------------

def _hadamard32_interleaved(v: np.ndarray) -> np.ndarray:
    """v fp16[..., 64] = one warp: lane t holds (v[2t], v[2t+1]); butterfly across lanes with fp16 adds in the
    exact order of cache_q.cuh:26-33 (for i=1,2,4,8,16: partner = lane^i; if lane&i: w=-w; w = w + partner)."""
    w = np.asarray(v, dtype=F16).reshape(v.shape[:-1] + (32, 2)).copy()
    lane = np.arange(32)
    i = 1
    while i < 32:
        pw = w[..., lane ^ i, :]
        neg = ((lane & i) != 0)[:, None]
        w = np.where(neg, -w, w).astype(F16)
        w = (w + pw).astype(F16)
        i <<= 1
    return w.reshape(v.shape)


def kv_pack_q4(x: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """x fp16[..., multiple of 64] (the reference works on 512-value blocks = 8 warps of 64; the math is per
    warp).  Returns (packed uint8[..., n/2], scales fp16[..., n/32]).  cache_q.cuh:4-78."""
    x = np.asarray(x, dtype=F16)
    shp = x.shape
    n = shp[-1]
    assert n % 64 == 0
    v = _hadamard32_interleaved(x.reshape(shp[:-1] + (n // 64, 64)))
    # absmax over lanes 0..15 / 16..31 of max(|lo|,|hi|)  -> 32 consecutive values
    g = np.abs(v).reshape(shp[:-1] + (n // 32, 32))
    amax = g.max(-1).astype(F16)
    with np.errstate(divide="ignore", invalid="ignore"):
        wn = (v.reshape(g.shape).astype(np.float64) / amax[..., None].astype(np.float64)).astype(F16)   # __h2div
    wq = (wn.astype(np.float64) * 8.0 + 8.0).astype(F16)                         # __hfma2(w, 8, 8)
    q = np.rint(wq.astype(np.float64))                                          # __half2int_rn (ties to even)
    q = np.where(np.isnan(q), 0, q)
    q = np.clip(q, 0, 15).astype(np.uint8).reshape(shp[:-1] + (n,))
    packed = (q[..., 0::2] | (q[..., 1::2] << 4)).astype(np.uint8)
    scales = (amax * F16(0.125)).astype(F16)
    return packed, scales


def kv_unpack_q4(packed: np.ndarray, scales: np.ndarray) -> np.ndarray:
    """cache_q.cuh:111-185: (q-8)*scale in fp16 -> Hadamard -> * 1/32."""
    p = np.asarray(packed, dtype=np.uint8)
    n = p.shape[-1] * 2
    q = np.empty(p.shape[:-1] + (n,), dtype=np.int32)
    q[..., 0::2] = p & 0xF
    q[..., 1::2] = p >> 4
    s = np.repeat(np.asarray(scales, dtype=F16), 32, axis=-1)
    w = ((q - 8).astype(F16) * s).astype(F16)
    v = _hadamard32_interleaved(w.reshape(w.shape[:-1] + (n // 64, 64))).reshape(w.shape)
    return (v * F16(1.0 / 32.0)).astype(F16)
