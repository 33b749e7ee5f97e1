"""Seeded synthetic EXL2 / GPTQ tensors in the reference's on-disk format (SURVEY.md 8d, Appendix B).

TEST INFRASTRUCTURE: used by tests/, bench.py and __graft_entry__.smoke() to make inputs.  It contains no
arithmetic of the hot path (packing only) -- the writer being mirrored is conversion/adaptivegptq.py:608-677
(`pack`) with exllamav2_ext/cuda/pack_tensor.cu:118-271 (`pack_columns`) and :10-36 (`pack_rows_4`).
"""
from __future__ import annotations

import math

import numpy as np


def pack_bitstream(q: np.ndarray, bits: int) -> np.ndarray:
    """q int[rows, N] with rows*bits % 32 == 0  ->  uint32[rows*bits/32, N], little-endian stream down the rows
    of each column (pack_columns_kernel, pack_tensor.cu:118-271)."""
    rows, N = q.shape
    assert (rows * bits) % 32 == 0
    R = rows * bits // 32
    out = np.zeros((R + 1, N), dtype=np.uint64)
    idx = np.arange(rows, dtype=np.int64) * bits
    wi = idx // 32
    sh = (idx % 32).astype(np.uint64)
    v = q.astype(np.uint64) << sh[:, None]
    np.bitwise_or.at(out, wi, v & np.uint64(0xFFFFFFFF))
    np.bitwise_or.at(out, wi + 1, v >> np.uint64(32))
    return out[:R].astype(np.uint32)


def group_plan(K: int, bits: list[int], bits_prop: list[float], group_size) -> list[tuple[int, int]]:
    """(bits, rows) per group.  conversion/qparams.py:73-84 / conversion/adaptivegptq.py:182-192,650."""
    if isinstance(group_size, int):
        group_size = {b: group_size for b in bits}
    elif isinstance(group_size, (list, tuple)):
        group_size = {b: g for b, g in zip(bits, group_size)}
    plan = []
    remaining = K
    for b, p in zip(bits, bits_prop):
        gsz = group_size[b]
        g = math.ceil(min(K * p, remaining) / gsz)
        for _ in range(g):
            rows = min(gsz, remaining)
            if rows <= 0:
                break
            plan.append((b, rows))
            remaining -= rows
    assert remaining <= 0, "bits_prop does not cover all rows"
    return plan


def make_exl2(K: int, N: int, bits=(4,), bits_prop=(1.0,), group_size=128, seed: int = 0, perm: bool = True,
              bias: bool = False, scale_max_range=(0.5, 4.0)) -> dict:
    """Synthetic EXL2 linear: uniform random q, random 4-bit group scales, q_scale_max ~ U(0.5, 4) (so the
    post-/256 scales are ~1e-2 like real checkpoints), seeded act-order permutation."""
    rng = np.random.default_rng(seed)
    assert N % 32 == 0 and K % 32 == 0
    plan = group_plan(K, list(bits), list(bits_prop), group_size)
    G = len(plan)
    strips = []
    q_groups = np.zeros((2 * G,), dtype=np.int16)
    qrow = 0
    for gi, (b, rows) in enumerate(plan):
        assert (rows * b) % 32 == 0
        q = rng.integers(0, 1 << b, size=(rows, N), dtype=np.int64)
        strips.append(pack_bitstream(q, b))
        q_groups[2 * gi] = b
        q_groups[2 * gi + 1] = qrow
        qrow += rows * b // 32
    q_weight = np.concatenate(strips, axis=0).astype(np.uint32).view(np.int32)
    nib = rng.integers(0, 16, size=(G, N), dtype=np.uint32)
    q_scale = np.zeros((G, N // 8), dtype=np.uint32)
    for i in range(8):
        q_scale |= nib[:, i::8] << np.uint32(4 * i)
    q_scale_max = rng.uniform(scale_max_range[0], scale_max_range[1], size=(G,)).astype(np.float16)
    w = {
        "q_weight": q_weight,
        "q_scale": q_scale.view(np.int32),
        "q_scale_max": q_scale_max,
        "q_groups": q_groups,
    }
    if perm:
        w["q_invperm"] = rng.permutation(K).astype(np.int32)
    else:
        w["q_invperm"] = np.arange(K, dtype=np.int32)
    if bias:
        w["bias"] = rng.normal(0, 0.1, size=(N,)).astype(np.float16)
    return w


def make_gptq(K: int, N: int, group_size: int = 128, seed: int = 0, act_order: bool = False, bias: bool = False) -> dict:
    """Synthetic GPTQ 4-bit linear (SURVEY.md 8d C1): uniform random nibbles, scales ~ U(0.002, 0.02),
    g_idx = arange//g, or a seeded permutation of it for act-order.  group_size <= 0: ungrouped (GPTQ's group_size -1),
    one group over all K rows and g_idx all zero -- with or without act-order, as such checkpoints ship."""
    rng = np.random.default_rng(seed)
    if group_size <= 0:
        group_size = K
    assert K % group_size == 0 and N % 8 == 0 and K % 8 == 0
    G = K // group_size
    q = rng.integers(0, 16, size=(K, N), dtype=np.int64)
    qweight = pack_bitstream(q, 4).view(np.int32)
    z = rng.integers(0, 16, size=(G, N), dtype=np.uint32)
    qzeros = np.zeros((G, N // 8), dtype=np.uint32)
    for i in range(8):
        qzeros |= z[:, i::8] << np.uint32(4 * i)
    scales = rng.uniform(0.002, 0.02, size=(G, N)).astype(np.float16)
    g_idx = (np.arange(K) // group_size).astype(np.int32)
    if act_order:
        g_idx = g_idx[rng.permutation(K)]
    w = {"qweight": qweight, "qzeros": qzeros.view(np.int32), "scales": scales, "g_idx": g_idx}
    if bias:
        w["bias"] = rng.normal(0, 0.1, size=(N,)).astype(np.float16)
    return w


def nbytes_algorithmic(w: dict, M: int = 1, accumulate: bool = False) -> int:
    """Algorithmic bytes of one linear call (SURVEY.md 8d): weights + scales (+perm u16) + a + c."""
    if "q_weight" in w:
        K = w["q_invperm"].shape[0]
        N = w["q_weight"].shape[1]
        b = w["q_weight"].nbytes + w["q_scale"].nbytes + w["q_scale_max"].nbytes + 2 * K
    else:
        K = w["qweight"].shape[0] * 8
        N = w["qweight"].shape[1]
        b = w["qweight"].nbytes + w["qzeros"].nbytes + w["scales"].nbytes
        if not (np.asarray(w["g_idx"]) == np.arange(K) // (K // w["qzeros"].shape[0])).all():
            b += 2 * K
    b += 2 * M * K + 2 * M * N * (2 if accumulate else 1)
    if "bias" in w:
        b += 2 * N
    return int(b)
