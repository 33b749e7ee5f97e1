"""The 8-bit K/V cache formats (Q6 = 8-bit keys + 4-bit values, Q8 = 8-bit keys and values): a numpy restatement of the
8-bit branch of the reference's cuda/cache_q.cuh, and the seeded cases of tests/golden/ref_kv_q68.npz
(written by tools/gen_golden_kv_q68.py from the reference extension).  The Q4 half of Q6 is exl2_oracle.kv_pack_q4."""
from __future__ import annotations

import hashlib

import numpy as np

import exl2_oracle as oracle

F16 = np.float16


def kv_pack_q8(x: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """x fp16[..., multiple of 64] -> (uint8[..., n] with value e at byte e, scales fp16[..., n/32]).  cache_q.cuh:78-108:
    the same Hadamard-32 and absmax as Q4, then w = w / absmax (__h2div), w * 128 + 128 (one __hfma2 rounding),
    q = clamp(rint(w), 0, 255), scale = absmax * half(1/128)."""
    x = np.asarray(x, dtype=F16)
    shp = x.shape
    n = shp[-1]
    assert n % 64 == 0
    v = oracle._hadamard32_interleaved(x.reshape(shp[:-1] + (n // 64, 64)))
    g = np.abs(v).reshape(shp[:-1] + (n // 32, 32))
    amax = g.max(-1).astype(F16)
    with np.errstate(divide="ignore", invalid="ignore"):
        wn = (v.reshape(g.shape).astype(np.float64) / amax[..., None].astype(np.float64)).astype(F16)   # __h2div
    wq = (wn.astype(np.float64) * 128.0 + 128.0).astype(F16)                     # __hfma2(w, 128, 128)
    q = np.rint(wq.astype(np.float64))                                          # __half2int_rn (ties to even)
    q = np.where(np.isnan(q), 0, q)
    q = np.clip(q, 0, 255).astype(np.uint8).reshape(shp[:-1] + (n,))
    scales = (amax * F16(1.0 / 128.0)).astype(F16)
    return q, scales


def kv_unpack_q8(packed: np.ndarray, scales: np.ndarray) -> np.ndarray:
    """cache_q.cuh:147-162 + :164-185: (q - 128) * scale in fp16 -> Hadamard -> * 1/32."""
    q = np.asarray(packed, dtype=np.uint8).astype(np.int32)
    n = q.shape[-1]
    s = np.repeat(np.asarray(scales, dtype=F16), 32, axis=-1)
    w = ((q - 128).astype(F16) * s).astype(F16)
    v = oracle._hadamard32_interleaved(w.reshape(w.shape[:-1] + (n // 64, 64))).reshape(w.shape)
    return (v * F16(1.0 / 32.0)).astype(F16)


def kv_unpack_exact(packed: np.ndarray, scales: np.ndarray, bits: int) -> np.ndarray:
    """The stored rows as the fused attention kernels read them: (code - offset) x scale and the inverse Hadamard-32 in fp64,
    with no rounding.  kv_unpack rounds every step to fp16, as the reference's q_to_fp16_kv does."""
    p = np.asarray(packed, dtype=np.uint8)
    if bits == 8:
        q = p.astype(np.float64) - 128.0
    else:
        q = np.empty(p.shape[:-1] + (p.shape[-1] * 2,), dtype=np.float64)
        q[..., 0::2], q[..., 1::2] = p & 0xF, p >> 4
        q -= 8.0
    n = q.shape[-1]
    w = (q * np.repeat(np.asarray(scales, dtype=np.float64), 32, axis=-1)).reshape(q.shape[:-1] + (n // 64, 32, 2))
    lane = np.arange(32)
    i = 1
    while i < 32:                   # the butterfly of oracle._hadamard32_interleaved, exact
        w = np.where(((lane & i) != 0)[:, None], -w, w) + w[..., lane ^ i, :]
        i <<= 1
    return w.reshape(q.shape) / 32.0


def widths(wbits: int) -> tuple[int, int]:
    """Element widths (keys, values) of a cache format."""
    return {4: (4, 4), 6: (8, 4), 8: (8, 8)}[wbits]


def kv_pack(x: np.ndarray, bits: int):
    return kv_pack_q8(x) if bits == 8 else oracle.kv_pack_q4(x)


def kv_unpack(packed: np.ndarray, scales: np.ndarray, bits: int) -> np.ndarray:
    return kv_unpack_q8(packed, scales) if bits == 8 else oracle.kv_unpack_q4(packed, scales)


def digest(a) -> np.ndarray:
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


# ---- the cases of ref_kv_q68.npz ----------------------------------------------------------------------------------
#   non-paged [batch, seq, heads, hd]: tokens [offset, offset + width) of every batch row, widened to 512-value blocks
#   paged     [pages, 256, heads, hd]: tokens [seqlen, seqlen + q_len) of every sequence through a permuted block table
NONPAGED = {
    "np512": dict(shape=(2, 5, 8, 64), offset=0, width=5, seed=11),         # dim 512
    "np512_off": dict(shape=(2, 6, 8, 64), offset=2, width=3, seed=12),     # a partial range
    "np256_off": dict(shape=(2, 8, 4, 64), offset=3, width=3, seed=13),     # dim 256: widened to tokens [2, 6)
}
PAGED = {
    "pg1024": dict(heads=8, hd=128, pages=4, block_table=[[2, 0], [3, 1]], seqlens=[250, 7], q_len=10, seed=21),  # crosses a page
    "pg256": dict(heads=2, hd=128, pages=4, block_table=[[1, 3], [0, 2]], seqlens=[251, 30], q_len=3, seed=22),    # dim 256: widens
}
PAGE = 256


def nonpaged_inputs(name):
    c = NONPAGED[name]
    rng = np.random.default_rng(c["seed"])
    k = rng.normal(0, 1, size=c["shape"]).astype(F16)
    v = rng.normal(0, 2, size=c["shape"]).astype(F16)
    return k, v


def paged_inputs(name):
    c = PAGED[name]
    rng = np.random.default_rng(c["seed"])
    shp = (c["pages"], PAGE, c["heads"], c["hd"])
    k = rng.normal(0, 1, size=shp).astype(F16)
    v = rng.normal(0, 2, size=shp).astype(F16)
    return k, v


def nonpaged_range(name) -> tuple[int, int]:
    """Token range the pack / unpack converts (ext_cache.cpp:150-157 widening)."""
    c = NONPAGED[name]
    dim = c["shape"][2] * c["shape"][3]
    offset, width = c["offset"], c["width"]
    if dim % 512:
        while (offset * dim) % 512:
            offset -= 1
        while (width * dim) % 512:
            width += 1
    return offset, offset + width


def paged_rows(name):
    """(sequence, token, page, row in page) of the tokens a paged pack converts: [seqlen, seqlen + q_len) widened to whole
    512-value blocks (cache.cu:177-184)."""
    c = PAGED[name]
    dim = c["heads"] * c["hd"]
    out = []
    for s, sl in enumerate(c["seqlens"]):
        a, b = sl * dim, (sl + c["q_len"]) * dim
        if dim % 512:
            a, b = a // 512 * 512, (b + 511) // 512 * 512
        for tok in range(a // dim, (b + dim - 1) // dim):
            pg = c["block_table"][s][tok // PAGE]
            out.append((s, tok, pg, tok % PAGE))
    return out
