"""The launch arithmetic of the fused K/V-cache decode attention (csrc/attn_q4.cu), restated in Python, and the fp64 truth the
GPU tests compare it with.

`plan()` restates the host side of `exl2b_paged_attn_decode_q` and the prologue of `attn_q4_kernel<HD, KB, VB>`: how many
CTAs share one (head, sequence), which positions each attends, how many of its cached rows sit in the staged window, and
whether the rest is read from global memory or streamed through the ring.  The GPU tests pick their sequence lengths and
needle positions from it, so they keep landing on the boundaries if a constant changes, and each asserts that the plan puts
it in the branch it claims to test.  tests/test_attn_regimes_plan.py pins the plan to the figures DESIGN.md §3.4 states.
"""
from __future__ import annotations

import numpy as np

import kv_q68

# attn_q4.cu: AQ_THREADS, AQ_WARPS, AQ_MAX_QLEN, AQ_SPLIT_MIN, AQ_SUB, AQ_RING, AQ_STAGE
AQ_THREADS = 256
AQ_WARPS = 8
AQ_MAX_QLEN = 8
AQ_SPLIT_MIN = 512
AQ_SUB = 128
AQ_RING = 4
AQ_STAGE = 512
SMEM_LIMIT = 200 * 1024           # attn_q4.cu AQ_SMEM_MAX (the host refusal and the kernels' attribute)
H100_SMS = 132
PAGE = 256


def widths(wbits: int) -> tuple[int, int]:
    return kv_q68.widths(wbits)


def smem_bytes(wbits: int, hd: int, q_len: int, max_ctx: int, nsplit: int, page_size: int = PAGE) -> dict:
    """Dynamic shared memory of one launch and the sizes it is made of (attn_q4.cu attn_launch_plan, attn_smem_map)."""
    kb, vb = widths(wbits)
    pps = max_ctx // page_size
    sc_len = max(AQ_SPLIT_MIN, (max_ctx + nsplit) // nsplit) + 8 if nsplit > 1 else max_ctx + q_len     # sc_len
    ring = max_ctx > 8192                                                                                 # ring_slots
    rowk, rowv, nsc = hd * kb // 8, hd * vb // 8, hd // 32
    window = AQ_STAGE // 2 if ring else AQ_STAGE
    stage = window * (hd + 4 * nsc) // (rowk + rowv + 4 * nsc) // 64 * 64                                 # stage
    sub = AQ_SUB * 4 // max(kb, vb)                                                                       # aq_sub
    smem = ((nsc * 36 + AQ_WARPS * hd + 2 * AQ_WARPS) * 4 + nsc * (80 + 8) + AQ_MAX_QLEN * (rowk + rowv)   # attn_smem_map total
            + 2 * AQ_MAX_QLEN * nsc * 2 + 2 * AQ_MAX_QLEN * hd * 4 + ((pps + 3) & ~3) * 4 + ((sc_len + 3) & ~3) * 4
            + stage * (rowk + rowv) + stage * nsc * 2 * 2 + (AQ_RING * sub * (max(rowk, rowv) + nsc * 2) if ring else 0))
    return dict(sc_len=sc_len, ring=ring, stage=stage, sub=sub, smem=smem, fits=smem <= SMEM_LIMIT)


def nsplit_of(q_len: int, max_ctx: int, H: int, B: int, sms: int = H100_SMS) -> int:
    """CTAs per (head, sequence) (attn_q4.cu attn_launch_plan, nsplit): split-KV only for one query over a cache above 1024 positions."""
    if q_len == 1 and max_ctx > 2 * AQ_SPLIT_MIN:
        by_ctx = (max_ctx + AQ_SPLIT_MIN - 1) // AQ_SPLIT_MIN
        by_sms = max(1, (2 * sms) // max(1, H * B))
        return max(1, min(by_ctx, by_sms, 16))
    return 1


def plan(wbits: int, hd: int, H: int, B: int, q_len: int, max_ctx: int, seqlens, sms: int = H100_SMS,
         page_size: int = PAGE) -> dict:
    """The launch `exl2b_paged_attn_decode_q` makes, and what each working CTA of it does.

    Returns nsplit, stage, ring, sub, sc_len, smem, fits, and `ctas`: one dict per (sequence b, split z) that works, with
      p_lo, p_hi   the positions it attends, [p_lo, p_hi) (query i of a CTA without split attends [0, seqlen + i + 1))
      c_hi         the end of its cached rows, [p_lo, c_hi)                                  (attn_q4.cu AttnCta::prologue)
      n_st         cached rows in the staged window, [p_lo, p_lo + n_st)                     (prologue)
      beyond       cached rows past the window, [p_lo + n_st, c_hi): from the ring if `ring`, else from global memory
      ntail        ring sub-chunks of SUB positions, from p_lo + n_st on                     (prologue, ring_pass)
      merge        it leaves a partial result for the merge (ns_act > 1)                     (end_query)
    A sequence whose seqlen + q_len exceeds max_ctx is refused by the kernel (prologue) and has no CTA here."""
    assert len(seqlens) == B
    nsplit = nsplit_of(q_len, max_ctx, H, B, sms)
    out = dict(nsplit=nsplit, **smem_bytes(wbits, hd, q_len, max_ctx, nsplit, page_size))
    out["ctas"] = []
    for b, seqlen in enumerate(seqlens):
        if seqlen < 0 or seqlen + q_len > max_ctx:
            continue
        ns_act, p_lo, p_hi = 1, 0, seqlen + q_len
        chunks = [(0, p_hi)]
        if nsplit > 1:
            n_all = seqlen + 1
            ns_act = min(nsplit, max(1, (n_all + AQ_SPLIT_MIN - 1) // AQ_SPLIT_MIN))
            chunk = (n_all + ns_act - 1) // ns_act
            chunks = [(z * chunk, min(n_all, z * chunk + chunk)) for z in range(ns_act)]
        for z, (p_lo, p_hi) in enumerate(chunks):
            c_hi = min(p_hi, seqlen)
            n_st = max(0, min(c_hi - p_lo, out["stage"]))
            beyond = max(0, c_hi - p_lo - n_st)
            ntail = (beyond + out["sub"] - 1) // out["sub"] if out["ring"] and beyond > 0 else 0
            out["ctas"].append(dict(b=b, z=z, seqlen=seqlen, ns_act=ns_act, p_lo=p_lo, p_hi=p_hi, c_hi=c_hi, n_st=n_st,
                                    beyond=beyond, ntail=ntail, merge=ns_act > 1))
    return out


def branches(p: dict, q_len: int, H: int, B: int, sms: int = H100_SMS) -> set:
    """The kernel branches a planned launch takes (the rows of the table in DESIGN.md §3.4)."""
    s = set()
    for c in p["ctas"]:
        if c["beyond"] > 0 and not p["ring"]:
            s.add("global")
        if c["ntail"] > 0:
            s.add("ring")
            if q_len > 1:
                s.add("ring_qlen")
        if c["merge"]:
            s.add("merge")
            if B > 1:
                s.add("merge_batch")
    if q_len == 1 and p["nsplit"] == 1 and H * B > sms and any(c["p_hi"] - c["p_lo"] > 2048 for c in p["ctas"]):
        s.add("batched")            # a cache long enough to split, but the batch fills the GPU: more CTAs than SMs, no split
    return s


def boundary_positions(p: dict, b: int, page_size: int = PAGE) -> list:
    """Cached positions of sequence b where a kernel goes wrong first: the edges of every CTA's window, of the first, second
    and last ring sub-chunk, of the rows read from global memory, of every split chunk, and of pages."""
    pos = set()
    seqlen = None
    for c in p["ctas"]:
        if c["b"] != b:
            continue
        seqlen = c["seqlen"]
        lo, st = c["p_lo"], c["p_lo"] + c["n_st"]
        pos.update({lo, lo + 1, st - 1, st, c["c_hi"] - 1, c["p_hi"] - 1, c["p_hi"]})
        for t in sorted({0, 1, c["ntail"] - 2, c["ntail"] - 1}):
            if 0 <= t < c["ntail"]:
                pos.update({st + t * p["sub"], st + t * p["sub"] + p["sub"] - 1})
    if seqlen is None:
        return []
    for e in range(page_size, seqlen + 1, page_size):
        if e == page_size or e + page_size > seqlen:
            pos.update({e - 1, e})
    pos.add(seqlen - 1)
    return sorted(x for x in pos if 0 <= x < seqlen)


# ---- fp64 truth -------------------------------------------------------------------------------------------------------

def gather_rows(cache_q, cache_s, block_table, b: int, seqlen: int, bits: int, page_size: int = PAGE) -> np.ndarray:
    """The first `seqlen` cached rows of sequence b, dequantised by the oracle: fp64 [seqlen, KVH, hd]."""
    p = np.arange(seqlen)
    pg, r = block_table[b, p // page_size], p % page_size
    return kv_q68.kv_unpack(cache_q[pg, r], cache_s[pg, r], bits).astype(np.float64)


def attention_truth(q, k_new, v_new, K_rows, V_rows, seqlens, softmax_scale: float, return_probs: bool = False):
    """fp64 softmax attention of every (sequence b, query i, head h): the dequantised cached rows K_rows[b] / V_rows[b]
    ([seqlen, KVH, hd]) followed by the UNQUANTISED new rows k_new / v_new, query i seeing positions [0, seqlen + i].
    Vectorised per kv head.  With return_probs, also the probabilities: probs[b] is [q_len, H, seqlen + q_len]."""
    B, q_len, H, hd = q.shape
    KVH = k_new.shape[2]
    g = H // KVH
    out = np.zeros((B, q_len, H, hd))
    probs = []
    for b in range(B):
        sl = seqlens[b]
        n = sl + q_len
        K = np.concatenate([K_rows[b], k_new[b].astype(np.float64)], 0)      # [n, KVH, hd]
        V = np.concatenate([V_rows[b], v_new[b].astype(np.float64)], 0)
        qb = q[b].astype(np.float64).reshape(q_len, KVH, g, hd)
        s = np.einsum("ikgd,nkd->ikgn", qb, K) * softmax_scale                # [q_len, KVH, g, n]
        mask = np.arange(n)[None, :] > (sl + np.arange(q_len))[:, None]       # causal among the new rows
        s = np.where(mask[:, None, None, :], -np.inf, s)
        pr = np.exp(s - s.max(-1, keepdims=True))
        pr /= pr.sum(-1, keepdims=True)
        out[b] = np.einsum("ikgn,nkd->ikgd", pr, V).reshape(q_len, H, hd)
        if return_probs:
            probs.append(pr.reshape(q_len, H, n))
    return (out, probs) if return_probs else out


def s_one_hot_row(hd: int, bits: int, e: int, neg: bool = False) -> np.ndarray:
    """The stored bytes of a row whose stored (rotated) values are zero except value e = +7 (or -8 with neg), at 4 and at 8
    bits.  With a scale of at most 8 significant bits, +7 * scale is exact in fp16, so the oracle's fp16 dequantisation of
    such a row is exact and a 40-nat score carries no rounding of the key into the truth."""
    if bits == 8:
        row = np.full(hd, 128, dtype=np.uint8)
        row[e] = 120 if neg else 135
    else:
        row = np.full(hd // 2, 0x88, dtype=np.uint8)
        nib = 0 if neg else 15
        row[e // 2] = (0x80 | nib) if e % 2 == 0 else (nib << 4 | 0x08)
    return row


def one_hot_amp(bits: int) -> int:
    return 7


def round8(x: float) -> np.float16:
    """x rounded to 8 significant bits, as fp16 (a scale whose products with -8..7 are exact in fp16)."""
    m, e = np.frexp(float(x))
    return np.float16(np.ldexp(np.round(m * 256) / 256, e))


def key_direction(hd: int, bits: int, e: int) -> np.ndarray:
    """The dequantised key of the stored one-hot e at scale 1, as fp64: +-7/32 on the 32 elements its Hadamard row covers."""
    row = s_one_hot_row(hd, bits, e)
    sc = np.ones(hd // 32, dtype=np.float16)
    return kv_q68.kv_unpack(row[None], sc[None], bits)[0].astype(np.float64)


def rotate_q_fp32(q_row: np.ndarray, scale_log2: np.float32) -> np.ndarray:
    """The kernel's fp32 query rotation (kv_format.cuh hadamard32_f, attn_q4.cu AttnCta::rotate_q): per 64-value unit, lane t holds elements (2t, 2t+1);
    butterfly w = fmaf(sign, w, partner) for i = 1..16; then * (scale_log2 * (1/32)).  Returns the rotated values in stored
    order [hd] (fp32)."""
    hd = q_row.shape[-1]
    f32 = np.float32
    w = q_row.astype(f32).reshape(hd // 64, 32, 2)
    lane = np.arange(32)
    i = 1
    while i < 32:
        pw = w[:, lane ^ i, :]
        sg = np.where((lane & i) != 0, f32(-1), f32(1))[None, :, None]
        w = (sg * w + pw).astype(f32)             # sg * w is exact: one rounding, as fmaf
        i <<= 1
    f = f32(f32(scale_log2) * f32(1.0 / 32.0))
    return (w.reshape(hd) * f).astype(f32)
