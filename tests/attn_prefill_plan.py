"""The launch arithmetic of the prompt attention over the quantised cache (csrc/attn_prefill.cu), restated in Python.

`smem_bytes()` restates prefill_smem_map, `grid()` the grid of exl2b_paged_attn_prefill_q and `appended_tokens()` which CTA
appends which new token.  tests/test_attn_prefill_plan.py pins them to the library (its refusal) and to DESIGN.md §3.8.
"""
from __future__ import annotations

import kv_q68

# attn_prefill.cu: AP_THREADS, AP_BM, AP_BN, AP_SMEM_MAX
AP_THREADS = 128
AP_BM = 64
AP_BN = 64
SMEM_LIMIT = 200 * 1024


def smem_bytes(wbits: int, hd: int, pages_per_seq: int) -> dict:
    """Dynamic shared memory of one CTA (prefill_smem_map) and the regions it is made of."""
    kb, vb = kv_q68.widths(wbits)
    nsc, rowk, rowv = hd // 32, hd * kb // 8, hd * vb // 8
    tiles = AP_BM * (hd + 8) * 2 + AP_BN * (hd + 8) * 2 + hd * (AP_BN + 8) * 2     # q, kh, vt (fp16)
    out = AP_BM * (hd + 4) * 4                                                      # fp32 output tile, over q / kh / vt
    raw = max(tiles, out)
    stage = AP_BN * (rowk + rowv + 2 * nsc * 2)
    total = raw + 2 * stage + ((pages_per_seq + 3) & ~3) * 4
    return dict(tiles=tiles, out=out, stage=stage, total=total, fits=total <= SMEM_LIMIT)


def max_pages(wbits: int, hd: int) -> int:
    """The largest page table a launch accepts."""
    fixed = smem_bytes(wbits, hd, 0)["total"]
    return (SMEM_LIMIT - fixed) // 16 * 4


def grid(q_len: int, H: int, KVH: int, B: int) -> tuple[int, int, int]:
    """(m-blocks, kv heads, sequences): a CTA owns AP_BM (token, head-in-group) rows of one kv head."""
    return ((q_len * (H // KVH) + AP_BM - 1) // AP_BM, KVH, B)


def appended_tokens(mb: int, q_len: int, group: int) -> range:
    """New tokens whose K / V units CTA m-block `mb` appends: those whose first row t * group lies in its rows."""
    m0 = mb * AP_BM
    return range((m0 + group - 1) // group, min(q_len, (m0 + AP_BM + group - 1) // group))


def key_tiles(seqlen: int, mb: int, q_len: int, group: int) -> int:
    """Key tiles a CTA walks: up to its last query's position (tiles wholly beyond it are skipped)."""
    rows = q_len * group
    t_hi = min(q_len - 1, (min(mb * AP_BM + AP_BM, rows) - 1) // group)
    return (seqlen + t_hi + 1 + AP_BN - 1) // AP_BN
