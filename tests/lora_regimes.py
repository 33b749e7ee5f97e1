"""The launch geometry of the LoRA kernel (csrc/lora.cu), restated in Python, and the case lists of the GPU tests that run it.

`launch()` restates `lora_launch` and the prologue of `lora_kernel`: how a cluster's CTAs split K, the dynamic shared memory
of the staged input rows, how warps share the stacked column groups of x·A, which CTA finishes which unit of output columns,
and whether a segment's rows of A are read 16 bytes at a time or element by element.  `regimes()` names the branches one
launch takes.  tests/test_gpu_lora_regimes.py parametrizes over the case lists below, and `case_launches()` turns each case
into the launches it makes, so tests/test_lora_regimes_plan.py can check on a machine without a GPU that together the cases
reach every branch, and the two cannot drift apart.
"""
from __future__ import annotations

import test_gpu_group_structures as _gs

# lora.cu: LORA_THREADS, LORA_WARPS, LORA_CLUSTER, LORA_MAX_CTAS, LORA_SMEM_MAX; lora.cuh: LORA_MT, LORA_MAX_RANK, LORA_MAX_SEGS
LORA_THREADS = 256
LORA_WARPS = 8
LORA_CLUSTER = 8
LORA_MAX_CTAS = 128
LORA_SMEM_MAX = 184 * 1024
LORA_MT = 8
LORA_MAX_RANK = 512
LORA_MAX_SEGS = 24

ADD, QKV, ACT_MUL = 0, 1, 2          # LoraEpilogue
NEOX, GPTJ = 2, 1                    # rope_style of make_q_attn

ATTN = ("q_proj", "k_proj", "v_proj", "o_proj")
MLP = ("gate_proj", "up_proj", "down_proj")
STAGES = {"qkv": ATTN[:3], "o": ATTN[3:], "gu": MLP[:2], "down": MLP[2:]}


def rank_slots(rank: int) -> int:
    """lora.cu:35: stacked columns of one segment, whole groups of 8"""
    return (rank + 7) & ~7


def kper(K: int) -> int:
    """lora.cu:49 / :341: K rows per cluster rank, ceil(K / 8) rounded up to a multiple of 8"""
    return ((K + LORA_CLUSTER - 1) // LORA_CLUSTER + 7) & ~7


def slices(K: int) -> list[tuple[int, int]]:
    """lora.cu:50: (k0, len) of each cluster rank; a rank past K has len 0"""
    kp = kper(K)
    out = []
    for cr in range(LORA_CLUSTER):
        k0 = min(K, cr * kp)
        out.append((k0, min(K, k0 + kp) - k0))
    return out


def smem_bytes(K: int, rows: int) -> int:
    """lora.cu:340-344: the fp32 input rows of one CTA's slice"""
    return min(LORA_MT, rows) * kper(K) * 4


def warps(R: int) -> dict:
    """lora.cu:85-87: column groups of 8, warps per group, and the warps that take no group"""
    groups = R >> 3
    wpg = 1 if groups >= LORA_WARPS else LORA_WARPS // groups
    idle = [w for w in range(LORA_WARPS) if w >= groups * wpg]
    work = {}
    for w in range(LORA_WARPS):
        if w in idle:
            continue
        work[w] = list(range(w // wpg, groups, LORA_WARPS // wpg))
    return dict(groups=groups, wpg=wpg, idle=idle, work=work)


def vec_load(rank: int, c0: int, k0: int, a_byte_offset: int) -> bool:
    """lora.cu:98-100: a column group reads A 16 bytes per row when it has 8 columns, the rank is a multiple of 8 and the group's
    first element of the slice is 16-byte aligned (a_byte_offset: A's address modulo 16)"""
    cnt = min(8, rank - c0)
    return cnt == 8 and rank % 8 == 0 and (a_byte_offset + 2 * (k0 * rank + c0)) % 16 == 0


def launch(epi: int, K: int, rows: int, n0: int = 0, heads_q: int = 0, heads_kv: int = 0, head_dim: int = 0) -> dict:
    """lora.cu:326-354 and :166-167: units of output columns, the grid, and each CTA's [u0, u1).  Raises ValueError where
    lora_launch refuses (odd output width on ADD; the staged slice above LORA_SMEM_MAX)."""
    if epi == QKV:
        unit_pairs, units = head_dim // 2, heads_q + 2 * heads_kv
    elif epi == ACT_MUL:
        unit_pairs, units = 64, (n0 + 63) // 64
    else:
        if n0 % 2:
            raise ValueError(f"LoRA: output width {n0} is odd")
        unit_pairs, units = 32, (n0 + 63) // 64
    tiles = (rows + LORA_MT - 1) // LORA_MT
    smem = smem_bytes(K, rows)
    if smem > LORA_SMEM_MAX:
        raise ValueError(f"LoRA: input width {K} needs {smem} bytes of shared memory per CTA")
    want = (units + LORA_CLUSTER - 1) // LORA_CLUSTER
    clusters = max(1, min(want, LORA_MAX_CTAS // LORA_CLUSTER // tiles))
    ctas = clusters * LORA_CLUSTER
    upc = (units + ctas - 1) // ctas
    cta_units = [(min(units, x * upc), min(units, x * upc + upc)) for x in range(ctas)]
    return dict(unit_pairs=unit_pairs, units=units, tiles=tiles, clusters=clusters, ctas=ctas, upc=upc, smem=smem,
                cta_units=cta_units, slices=slices(K))


def columns(epi: int, u: int, i: int, n0: int = 0, head_dim: int = 0, heads_q: int = 0, heads_kv: int = 0, sincos: int = 0,
            neox: bool = True, rope: bool = True):
    """lora.cu:168-200: the (projection, column) pair a thread of unit u, pair i finishes, and whether it rotates them; None for
    a pair past N"""
    idx = u * (head_dim // 2 if epi == QKV else 64 if epi == ACT_MUL else 32) + i
    if epi == QKV:
        h, pa = u, 0
        if h >= heads_q:
            h, pa = h - heads_q, 1
        if pa == 1 and h >= heads_kv:
            h, pa = h - heads_kv, 2
        rot = rope and pa < 2
        S2 = sincos // 2
        if rot and neox:
            if i < S2:
                ca, cb = i, i + S2
            else:
                ca, cb, rot = sincos + 2 * (i - S2), sincos + 2 * (i - S2) + 1, False
        else:
            ca, cb = 2 * i, 2 * i + 1
            rot = rot and ca < sincos
        return (pa, ca + h * head_dim), (pa, cb + h * head_dim), rot
    if epi == ACT_MUL:
        return ((0, idx), (1, idx), False) if idx < n0 else None
    return ((0, 2 * idx), (0, 2 * idx + 1), False) if 2 * idx < n0 else None


# ---- the blocks the GPU tests build ----------------------------------------------------------------------------------------------
# name: hidden, heads, kv heads, head dim, intermediate, rope style, rotary width (sincos_size)
BLOCKS = {
    "hd64": (512, 8, 2, 64, 1408, NEOX, 64),           # test_gpu_lora's hd64-gqa-neox shapes
    "s80": (160, 4, 2, 80, 480, NEOX, 32),             # hidden 160: empty K slices on q|k|v and gate|up; 480: short slice,
    "s96": (160, 2, 1, 96, 480, GPTJ, 48),             # N tails on gate|up (480) and down (160); partial rotary widths
    "s128": (160, 2, 1, 128, 480, GPTJ, 128),
    "s256": (160, 2, 1, 256, 480, NEOX, 128),
    "k1376": (1376, 8, 4, 64, 1376, NEOX, 64),         # test_gpu_group_structures' exl2_4b_g128_k1376 format
    "70b": (8192, 64, 8, 128, 28672, NEOX, 128),       # one Llama-2-70B layer: K = 28672 on down
}
# the 14 group formats of test_gpu_group_structures: name -> (hidden, intermediate), with its heads and head dim
FORMAT_SHAPES = {name: (v[1], v[2]) for name, v in _gs.FORMATS.items()}


def block_shape(block: str) -> tuple:
    if block.startswith("fmt:"):
        hid, inter = FORMAT_SHAPES[block[4:]]
        return (hid, _gs.HEADS, _gs.KV_HEADS, _gs.HD, inter, NEOX, _gs.HD)
    return BLOCKS[block]


# ---- adapter sets: [(id, {projection: rank})] ----------------------------------------------------------------------------------

def uniform(rank: int, targets=ATTN + MLP, key: int = 1) -> list:
    return [(key, {t: rank for t in targets})]


ODD = [(1, {p: 3 for p in ATTN + MLP}), (2, {"q_proj": 12, "v_proj": 33, "o_proj": 1, "gate_proj": 12, "up_proj": 100,
                                            "down_proj": 33})]
DOWN_ONLY = [(3, {"down_proj": 37})]


def stacked(stage: str, R: int) -> list:
    """adapters whose segments on `stage` stack to exactly R columns; R = 512 is the stage bound: 24 segments of ranks that are not
    multiples of 8 on q|k|v (8 adapters x 3 projections), 16 on gate|up, 8 of rank 64 on o and down"""
    projs = STAGES[stage]
    if R == 512:
        if stage == "qkv":
            return [(10 + i, {"q_proj": 17 + i, "k_proj": 9 + (i % 7), "v_proj": 24 - i}) for i in range(8)]
        if stage == "gu":
            return [(10 + i, {"gate_proj": 25 + i, "up_proj": 32 - i}) for i in range(8)]
        return [(10 + i, {projs[0]: 64}) for i in range(8)]
    # smaller widths: 8-column groups spread over the stage's projections and two adapters, the first with an odd rank
    groups = R // 8
    ads = {10: {}, 11: {}}
    for g in range(groups):
        key, p = 10 + g % 2, projs[(g // 2) % len(projs)]
        ads[key][p] = ads[key].get(p, 0) + 8
    first = next(iter(ads[10]))
    ads[10][first] -= 3                         # 3 fewer: the same columns, one scalar-loaded group
    return [(k, v) for k, v in ads.items() if v]


def set_launches(block: str, adapters: list, rows: int, active=None, misaligned: int = 0, norm: bool = True) -> list:
    """The LoRA launches one pass of the attention and MLP blocks makes with `adapters` registered and `active` (default: all)
    ids forwarded: dicts of launch() arguments plus the stacked ranks, rope and A alignment"""
    hid, H, KVH, hd, inter, style, rot = block_shape(block)
    ids = [k for k, _ in adapters] if active is None else active
    by_id = dict(adapters)
    out = []
    stages = (("qkv", QKV, hid, H * hd), ("o", ADD, H * hd, hid), ("gu", ACT_MUL, hid, inter), ("down", ADD, inter, hid))
    for st, epi, K, N in stages:
        ranks = [by_id[i][p] for i in ids if i in by_id for p in STAGES[st] if p in by_id[i]]   # lora_stack order
        if not ranks:
            continue
        out.append(dict(stage=st, epi=epi, K=K, rows=rows, n0=N, heads_q=H, heads_kv=KVH, head_dim=hd, ranks=ranks,
                        rope=style if epi == QKV else 0, sincos=rot, misaligned=misaligned))
    return out


def regimes(l: dict) -> set:
    """the branches of lora_kernel one launch takes"""
    g = launch(l["epi"], l["K"], l["rows"], l["n0"], l["heads_q"], l["heads_kv"], l["head_dim"])
    R = sum(rank_slots(r) for r in l["ranks"])
    w = warps(R)
    out = {f"wpg{w['wpg']}"}
    if w["idle"]:
        out.add(f"idle_warps_g{w['groups']}")
    lens = [n for _, n in g["slices"]]
    if 0 in lens:
        out.add("empty_slice")
    if any(0 < n < kper(l["K"]) for n in lens):
        out.add("short_slice")
    for r in l["ranks"]:
        for c0 in range(0, r, 8):
            for k0, n in g["slices"]:
                if n and not vec_load(r, c0, k0, l["misaligned"]):
                    out.add("scalar_misaligned" if r % 8 == 0 else "scalar_odd_rank")
    if R == LORA_MAX_RANK and len(l["ranks"]) == LORA_MAX_SEGS:
        out.add("R512_24segs")
    if R == LORA_MAX_RANK:
        out.add(f"R512_{l['stage']}")
    if g["tiles"] > LORA_MAX_CTAS // LORA_CLUSTER:
        out.add("tiles_gt_16")
    if g["tiles"] > 1 and l["rows"] % LORA_MT:
        out.add("partial_last_tile")
    if l["epi"] != QKV and l["n0"] % 64:
        out.add("n_tail_add" if l["epi"] == ADD else "n_tail_act_mul")
    if l["epi"] == QKV and l["rope"] and l["sincos"] < l["head_dim"]:
        out.add("neox_partial" if l["rope"] == NEOX else "gptj_partial")
    if g["smem"] > 100 * 1024:
        out.add("slice_gt_100KB")
    return out


# every branch the GPU cases must reach between them
REQUIRED = {"empty_slice", "short_slice", "wpg1", "wpg2", "wpg4", "wpg8", "idle_warps_g3", "idle_warps_g5", "idle_warps_g7",
            "scalar_odd_rank", "scalar_misaligned", "R512_24segs", "R512_qkv", "R512_o", "R512_gu", "R512_down", "tiles_gt_16",
            "partial_last_tile", "n_tail_add", "n_tail_act_mul", "neox_partial", "gptj_partial", "slice_gt_100KB"}


# ---- the GPU case lists (tests/test_gpu_lora_regimes.py) ----------------------------------------------------------------------

ODD_RANKS = (1, 3, 12, 33, 100)
PADDED_CASES = [(r, rows) for r in ODD_RANKS for rows in (1, 8, 40)]           # odd rank == zero-padded rank, bit for bit
MISALIGNED_CASES = [(off, rows) for off, rows in ((1, 1), (3, 8), (5, 40), (7, 17))]   # A at an element offset, rank 16

# (block, rope style, rotary width, rows, past_len): B = 0 bit-identical to the call without adapters; past_len -1 takes each
# sequence's position from past_lens, >= 0 adds it
ZERO_B_CASES = (
    [("hd64", s, w, rows, past) for s in (NEOX, GPTJ) for w in (64, 32) for rows in (1, 8, 17, 40) for past in (-1, 6)]
    + [("s80", s, w, rows, -1) for s in (NEOX, GPTJ) for w in (80, 32) for rows in (1, 8, 17, 40)]
    + [("s96", GPTJ, 48, rows, 3) for rows in (1, 8, 40)] + [("s96", NEOX, 96, rows, -1) for rows in (8, 17)]
    + [("s128", s, w, rows, -1) for s in (NEOX, GPTJ) for w in (128, 64) for rows in (1, 8, 40)]
    + [("s256", s, w, rows, 2) for s in (NEOX, GPTJ) for w in (256, 128) for rows in (1, 8, 17)]
    + [("fmt:exl2_4b_g256", NEOX, 64, 2, -1), ("fmt:gptq_g512_act", NEOX, 64, 2, 4)]
)

FORMAT_ROWS = (1, 2, 8, 9, 16, 17, 40)
FORMAT_CASES = [(f, rows, s) for f in FORMAT_SHAPES for rows in FORMAT_ROWS for s in ("odd", "down")]
OWN_PERM_CASES = list(FORMAT_SHAPES)                      # q/k/v and gate/up on their own permutations, one row

GEOMETRY_CASES = [(b, rows) for b in ("s80", "s96", "s256", "k1376") for rows in (1, 8, 17, 40)]

STACK_WIDTHS = (8, 16, 24, 40, 56, 512)
STACK_CASES = [(st, R, rows) for st in STAGES for R in STACK_WIDTHS for rows in (1, 9, 40)]

LONG_ROWS = ((129, 3), (256, 4), (1000, 8))                # (rows, sequences)
FULL_ROWS = (1, 8, 40)
OPTION_CASES = [(opt, rows) for opt in ("no_norm", "no_residual") for rows in (1, 8, 40)]

DECODER_ROWS = 2 * 96                                     # prefill_rows at 2 x 96: 24 row tiles
DECODER_ADAPTERS = [(12, ATTN + MLP), (33, ("q_proj", "v_proj"))]


def case_launches() -> dict:
    """every GPU case list as the launches it makes: list name -> [launch dict]"""
    odd = lambda r: uniform(r)
    out = {}
    out["padded"] = [l for r, rows in PADDED_CASES for l in set_launches("hd64", odd(r), rows)]
    out["misaligned"] = [l for off, rows in MISALIGNED_CASES for l in set_launches("hd64", uniform(16), rows, misaligned=2 * off)]
    out["zero_b"] = []
    for block, style, w, rows, _ in ZERO_B_CASES:
        for l in set_launches(block, ODD, rows):
            if l["epi"] == QKV:
                l.update(rope=style, sincos=w)
            out["zero_b"].append(l)
    out["formats"] = [l for f, rows, s in FORMAT_CASES for l in set_launches("fmt:" + f, ODD if s == "odd" else DOWN_ONLY, rows)]
    out["own_perm"] = [l for f in OWN_PERM_CASES for l in set_launches("fmt:" + f, ODD, 1)]
    out["geometry"] = [l for b, rows in GEOMETRY_CASES for l in set_launches(b, ODD, rows)]
    out["stacked"] = []
    for st, R, rows in STACK_CASES:
        ads = stacked(st, R)
        active = [k for k, _ in ads][::-1] + [999]
        out["stacked"] += set_launches("hd64", ads, rows, active=active)
    out["long"] = [l for rows, _ in LONG_ROWS for l in set_launches("hd64", ODD, rows)]
    out["full"] = [l for rows in FULL_ROWS for l in set_launches("70b", uniform(16), rows)]
    out["options"] = [l for _, rows in OPTION_CASES for l in set_launches("hd64", ODD, rows)]
    return out
