"""Synthetic checkpoints generated directly on the GPU in the reference's on-disk tensor format (EXL2 / GPTQ).

There is no network, hence no real weights: bench.py and the decode model use random-bit tensors of the exact
shapes/dtypes a converted model has (SURVEY.md 8d, Appendix B).  A uniformly random bit stream IS a uniformly
random q for every bit width, so q_weight is just random int32 words; group tables follow
conversion/qparams.py:73-84 (the converter's group plan).
"""
from __future__ import annotations

import math

import torch


def group_plan(K: int, bits, bits_prop, group_size) -> list[tuple[int, int]]:
    if isinstance(group_size, int):
        group_size = {b: group_size for b in bits}
    elif isinstance(group_size, (list, tuple)):
        group_size = {b: g for b, g in zip(bits, group_size)}
    plan, remaining = [], K
    for b, p in zip(bits, bits_prop):
        gsz = group_size[b]
        g = math.ceil(min(K * p, remaining) / gsz)
        for _ in range(g):
            rows = min(gsz, remaining)
            if rows <= 0:
                break
            plan.append((b, rows))
            remaining -= rows
    assert remaining <= 0
    return plan


def random_exl2(K: int, N: int, bits=(4,), bits_prop=(1.0,), group_size=128, device="cuda:0", seed: int = 0,
                perm: bool = True, weight_std: float | None = None, perm_seed: int | None = None) -> dict:
    """Random EXL2 tensors.  weight_std: nominal standard deviation of the dequantised weights -- the realised one is
    ~1.4x larger because scale nibbles are uniform, see tests/test_synthetic.py -- (1/sqrt(K) keeps a
    random-init network's activations O(1), like a trained checkpoint's ~0.02 at K = 4096); None: scale_max in
    [0.5, 4) stored units, i.e. weights of magnitude ~5 (fine for single-matrix tests, overflows fp16 in a deep stack)."""
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    plan = group_plan(K, list(bits), list(bits_prop), group_size)
    G = len(plan)
    q_groups = torch.zeros((2 * G,), dtype=torch.int16)
    qrow = 0
    for gi, (b, rows) in enumerate(plan):
        q_groups[2 * gi] = b
        q_groups[2 * gi + 1] = qrow
        qrow += rows * b // 32
    w = {
        "q_weight": torch.randint(-2**31, 2**31 - 1, (qrow, N), dtype=torch.int32, device=device, generator=gen),
        "q_scale": torch.randint(-2**31, 2**31 - 1, (G, N // 8), dtype=torch.int32, device=device, generator=gen),
        "q_scale_max": (torch.rand((G,), device=device, generator=gen) * 3.5 + 0.5).half(),
        "q_groups": q_groups.to(device),
        "q_invperm": (torch.randperm(K, device=device, generator=gen) if perm else torch.arange(K, device=device)).to(torch.int32),
    }
    if perm and perm_seed is not None:
        # matrices quantised against the same input share one activation-order permutation (conversion/quantize.py:138-139)
        pg = torch.Generator(device=device)
        pg.manual_seed(0x5EED0000 + perm_seed)
        w["q_invperm"] = torch.randperm(K, device=device, generator=pg).to(torch.int32)
    if weight_std is not None:
        # std of (q - 2^(b-1)) for uniform q is 2^b / sqrt(12); E[(s+1)^2] for a uniform 4-bit scale nibble is 93.5;
        # the stored q_scale_max carries a factor 256 (the loader multiplies by 1/256, ext.py:336 of the reference)
        b = torch.tensor([p[0] for p in plan], dtype=torch.float32, device=device)
        jitter = torch.rand((G,), device=device, generator=gen) * 0.6 + 0.7
        w["q_scale_max"] = (256.0 * weight_std / ((2.0 ** b) / math.sqrt(12.0) * 93.5) * jitter).half()
    w["q_perm"] = torch.argsort(w["q_invperm"]).to(torch.int)
    return w


def random_gptq(K: int, N: int, group_size: int = 128, device="cuda:0", seed: int = 0, act_order: bool = False,
                weight_std: float | None = None, perm_seed: int | None = None) -> dict:
    """Random GPTQ 4-bit tensors.  weight_std: standard deviation of the dequantised weights (std of q - zero for uniform
    nibbles is ~6.5); None: scales ~ U(0.002, 0.02) as in SURVEY.md 8d C1.  perm_seed: matrices quantised against the same
    input share their act-order g_idx.  group_size <= 0: ungrouped (GPTQ's group_size -1), one group and g_idx all zero."""
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    if group_size <= 0:
        group_size = K
    G = K // group_size
    g_idx = (torch.arange(K) // group_size).to(torch.int32)
    if act_order:
        g_idx = g_idx[torch.randperm(K, generator=torch.Generator().manual_seed(seed if perm_seed is None else 0x5EED0000 + perm_seed))]
    scales = torch.rand((G, N), device=device, generator=gen) * 0.018 + 0.002
    if weight_std is not None:
        scales = scales * (weight_std / (0.011 * 6.5))
    return {
        "qweight": torch.randint(-2**31, 2**31 - 1, (K // 8, N), dtype=torch.int32, device=device, generator=gen),
        "qzeros": torch.randint(-2**31, 2**31 - 1, (G, N // 8), dtype=torch.int32, device=device, generator=gen),
        "scales": scales.half(),
        "g_idx": g_idx,
    }


def random_linear(K: int, N: int, plan, device="cuda:0", seed: int = 0, weight_std: float | None = None, perm_seed: int | None = None) -> dict:
    """plan = (bits, bits_prop, group_size) for EXL2, or ("gptq", group_size, act_order)."""
    if plan[0] == "gptq":
        return random_gptq(K, N, plan[1], device, seed, act_order=plan[2], weight_std=weight_std, perm_seed=perm_seed)
    bits, prop, gs = plan
    return random_exl2(K, N, bits, prop, gs, device=device, seed=seed, weight_std=weight_std, perm_seed=perm_seed)


def algorithmic_bytes(w: dict, M: int = 1, accumulate: bool = False) -> int:
    """Bytes a linear call must move (SURVEY.md 8d): packed weights + scales (+ u16 perm) + a + c."""
    if "q_weight" in w:
        K, N = w["q_invperm"].shape[0], w["q_weight"].shape[1]
        b = w["q_weight"].numel() * 4 + w["q_scale"].numel() * 4 + w["q_scale_max"].numel() * 2 + 2 * K
    else:
        K, N = w["qweight"].shape[0] * 8, w["qweight"].shape[1]
        b = w["qweight"].numel() * 4 + w["qzeros"].numel() * 4 + w["scales"].numel() * 2
        if "q_perm" in w or ("g_idx" in w and not bool((w["g_idx"][:-1] <= w["g_idx"][1:]).all())):
            b += 2 * K
    return b + 2 * M * K + 2 * M * N * (2 if accumulate else 1)
