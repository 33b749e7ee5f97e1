"""Rows past a sequence's length never reach its output, kernel by kernel: every cache row at or past each sequence's length,
and every row of a page no sequence owns, holds random codes at the poison scale of decoder_truth.poison_past (dequantised
elements up to ~2^12), so that in every head about half of them score thousands of nats above any live row.  A mask that
lets one such row into a max, a sum or P V moves the output by O(10^3); with ordinary random rows past the length the same
slip moves it by ~1/n and hides under the tolerance at the thousands of positions most regime tests use.

Each kernel's output is compared with the fp64 truth over the live rows only (attn_regimes.attention_truth, the tolerance of
the kernel's own tests), and every byte outside the rows the launch appends is checked unchanged, poison included.

  paged_attn_decode_q4 (csrc/attn_q4.cu), Q4 / Q6 / Q8 at hd 64 and 128, lengths from the plan restatements
  (tests/attn_regimes.py, tests/attn_long_plan.py) put at every edge where a mask decides:
    short        the warp-local pass: lengths whose own warp partition ends a range at the length (_warp_end_lengths)
    global_q1    q_len 1, no split: the staged window's end n_st - 1, n_st, n_st + 1, page ends
    global_qlen  q_len 4: the same with four new rows, one sequence ending at the capacity, appends across a page end
    split        split-KV merge, B = 8: lengths where a sequence gains a chunk (n_all = seqlen + 1 at multiples of 512 +- 1)
    ring         split-KV with the ring: the last chunk's rows past the window end at a ring sub-chunk end, +- 1
    ring_qlen    q_len 2, no split, the ring: the same edges with two new rows
    batched      32 heads over 8, B = 9: more CTAs than SMs, no split
    passes       32 heads over 8, B = 9, one page above the single-pass bound: lengths at pass ends +- 1
  paged_attn_prefill_q (csrc/attn_prefill.cu): lengths at the 64-position key tile ends and page ends, 70 new rows
  attn_decode.cu (the fp16 reference attention): fp16 rows past the length at +-2^12
  q_to_fp16_kv / fp16_to_q_kv: no temp row past a length is written, no cache byte outside [seqlen, seqlen + q_len)
Each decode case asserts the branches its lengths are chosen for, from the plan."""
import math
import zlib

import numpy as np
import pytest
import torch

import attn_long_plan as alp
import attn_regimes as ar
import decoder_truth as dt
import kv_q68
import test_gpu_attn_prefill as tp
import test_gpu_attn_regimes as rg
import test_gpu_attn_short_path as sp

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FMTS = rg.FMTS
PAGE = ar.PAGE


def seed_of(*key):
    return zlib.crc32(repr(key).encode())


def edges(*xs):
    return sorted({v for x in xs for v in (x - 1, x, x + 1)})


def _ring_edges(wbits, hd, H, B, max_ctx, lo, want):
    """Lengths from lo on whose last split chunk (at batch B) has its rows past the staged window end exactly at a ring
    sub-chunk end, one row before it and one after it."""
    out = {}
    for s in range(lo, max_ctx):
        p = ar.plan(wbits, hd, H, B, 1, max_ctx, [s] * B)
        last = [c for c in p["ctas"] if c["b"] == 0][-1]
        r = last["beyond"] % p["sub"]
        if last["beyond"] > p["sub"] and r in (0, 1, p["sub"] - 1) and r not in out:
            out[r] = s
            if len(out) == want:
                break
    return sorted(out.values())


def _warp_end_lengths(hd, st):
    """Lengths whose own warp partition of the short path (attn_q4.cu AttnCta::staged_pass: 8 warps, each a contiguous range
    of whole steps of g = 32 / (hd / 32) positions over [0, seqlen + 1)) puts the length at a range end: seqlen + 1 an exact
    multiple of 8 g (every warp full, the new row the last of the last warp), the last warp holding the new row alone, and the
    last warp left empty."""
    g = 32 // (hd // 32)
    kinds = {}
    for s in range(2, st):
        n = s + 1
        per = -(-n // (ar.AQ_WARPS * g)) * g
        used = -(-n // per)
        last = n - (used - 1) * per
        kind = "full" if n % (ar.AQ_WARPS * g) == 0 else "one" if last == 1 else "empty" if used < ar.AQ_WARPS else None
        if kind and kinds.get(kind, (0, []))[0] < 2:
            c, v = kinds.get(kind, (0, []))
            kinds[kind] = (c + 1, v + [s])
    return sorted(x for _, v in kinds.values() for x in v)


def case_of(name, wbits, hd):
    """(H, KVH, q_len, max_ctx, seqlens, branches the launch must take)."""
    st = ar.smem_bytes(wbits, hd, 1, 1024, 1)["stage"]
    if name == "short":
        return 8, 2, 1, 1024, [0, 1] + _warp_end_lengths(hd, st) + [st - 1], {"short"}
    if name == "global_q1":
        return 8, 8, 1, 1024, edges(st) + [255, 256, 257, 1023], {"global"}
    if name == "global_qlen":
        return 8, 2, 4, 4096, edges(st) + [254, 4092], {"global"}
    if name == "split":
        return 8, 2, 1, 4096, [0, 1, 511, 512, 513, 1023, 1024, 4095], {"merge_batch"}
    if name == "ring":
        return 8, 8, 1, 16384, [16383] + _ring_edges(wbits, hd, 8, 4, 16384, 9000, 3), {"ring", "merge_batch"}
    if name == "ring_qlen":
        rst = ar.smem_bytes(wbits, hd, 2, 12288, 1)["stage"]
        sub = ar.smem_bytes(wbits, hd, 2, 12288, 1)["sub"]
        return 8, 8, 2, 12288, [rst + 40 * sub - 1, rst + 40 * sub, rst + 40 * sub + 1, 40 * 256 - 1, 12286], {"ring_qlen"}
    if name == "batched":
        return 32, 8, 1, 4096, [0, 1, 255, 256, 257, st - 1, st, st + 1, 4095], {"batched", "global"}
    if name == "passes":
        cap = alp.largest_fit(wbits, hd, 32, 9) + PAGE
        pl = alp.long_plan(wbits, hd, 32, 9, 1, cap)["pass_len"]
        return 32, 8, 1, cap, [0, 1, 256, 257, 303, pl - 1, pl, pl + 1, cap - 1], {"passes"}
    raise KeyError(name)


NAMES = ["short", "global_q1", "global_qlen", "split", "ring", "ring_qlen", "batched", "passes"]


def poison_cache(rng, kq, ks, vq, vs, bt, seqlens, kb, vb):
    """Poison every row of kq / ks / vq / vs ([pages, PAGE, KVH, ...]) at or past each length, and every unowned page."""
    mask = np.ones(kq.shape[:2], dtype=bool)
    for b, sl in enumerate(seqlens):
        p = np.arange(sl)
        mask[bt[b][p // PAGE], p % PAGE] = False
    n = int(mask.sum())
    for q, s, bits in ((kq, ks, kb), (vq, vs, vb)):
        pq, ps = dt.poison_rows(rng, (n,) + q.shape[2:], (n,) + s.shape[2:], bits)
        q[mask], s[mask] = pq, ps
    return mask


def build(name, wbits, hd):
    H, KVH, q_len, max_ctx, seqlens, expect = case_of(name, wbits, hd)
    seqlens = [s for s in seqlens if 0 <= s <= max_ctx - q_len]
    B, pps, group = len(seqlens), max_ctx // PAGE, H // KVH
    kb, vb = ar.widths(wbits)
    lp = alp.long_plan(wbits, hd, H, B, q_len, max_ctx, seqlens)
    p = ar.plan(wbits, hd, H, B, q_len, max_ctx, seqlens)
    got = ar.branches(p, q_len, H, B) | ({"passes"} if lp["passes"] else set()) | ({"short"} if q_len == 1 and sp.staged(p) else set())
    assert expect <= got, (name, expect, got)
    assert lp["fits"]
    rng = np.random.default_rng(seed_of(name, wbits, hd))
    pages_total = B * pps + 1                                   # one page no sequence owns
    bt = rng.permutation(pages_total)[:B * pps].reshape(B, pps).astype(np.int32)
    shp = (pages_total, PAGE, KVH)
    kq = rng.integers(0, 256, size=shp + (hd * kb // 8,), dtype=np.uint8)
    vq = rng.integers(0, 256, size=shp + (hd * vb // 8,), dtype=np.uint8)
    ks = (rng.uniform(0.05, 0.15, size=shp + (hd // 32,)) / (16 if kb == 8 else 1)).astype(np.float16)
    vs = (rng.uniform(0.02, 0.3, size=shp + (hd // 32,)) / (16 if vb == 8 else 1)).astype(np.float16)
    poison_cache(rng, kq, ks, vq, vs, bt, seqlens, kb, vb)
    c = dict(H=H, KVH=KVH, q_len=q_len, max_ctx=max_ctx, seqlens=seqlens, B=B, group=group, sigma=1.0 / math.sqrt(hd),
             beta=rg.BETA, bt=bt, kq=kq, ks=ks, vq=vq, vs=vs, kb=kb, vb=vb, needles=[], plan=lp)
    return c, rng


DECODE_CASES = [(w, hd, n) for (w, hd) in FMTS for n in NAMES]


@pytest.mark.parametrize("wbits,hd,name", DECODE_CASES, ids=[f"q{w}-hd{hd}-{n}" for w, hd, n in DECODE_CASES])
def test_decode_past_length(wbits, hd, name):
    c, rng = build(name, wbits, hd)
    K, V = rg._rows(c, c["kq"], c["ks"], c["vq"], c["vs"])
    q, kn, vn = rg.make_inputs(c, "random", rng, hd)
    rg.run_case(c, wbits, hd, q, kn, vn, c["kq"], c["ks"], c["vq"], c["vs"], K, V, ("past_length", name, wbits, hd))
    if name == "short":           # the warp-local pass ran where the plan says
        n = sp.debug_counter(lambda: rg.launch(c, q, kn, vn, c["kq"], c["ks"], c["vq"], c["vs"]))
        assert n == len(sp.staged(ar.plan(wbits, hd, c["H"], c["B"], 1, c["max_ctx"], c["seqlens"]))) * c["H"]


# ---- prompt attention over the quantised cache --------------------------------------------------------------------------------

PREFILL_LENS = [0, 1, 63, 64, 65, 127, 128, 255, 256, 257]


@pytest.mark.parametrize("wbits,hd", FMTS)
def test_prefill_past_length(wbits, hd):
    c = tp.make_case(wbits, hd, 8, 2, PREFILL_LENS, 70, seed=seed_of("prefill", wbits, hd) % 1000, spare_pages=2)
    rng = np.random.default_rng(seed_of("prefill-poison", wbits, hd))
    mask = poison_cache(rng, c["kq"], c["ks"], c["vq"], c["vs"], c["bt"], c["seqlens"], c["kb"], c["vb"])
    out, kq, ks, vq, vs = tp.launch(c)
    torch.cuda.synchronize()
    assert np.isfinite(out.float().cpu().numpy()).all()
    tp.compare(c, out, "past_length")
    for b, sl in enumerate(c["seqlens"]):             # the appended rows leave the poison
        p = np.arange(sl, sl + c["q_len"])
        mask[c["bt"][b][p // PAGE], p % PAGE] = False
    for got, want, what in ((kq, c["kq"], "k"), (ks, c["ks"], "k scales"), (vq, c["vq"], "v"), (vs, c["vs"], "v scales")):
        g = got.cpu().numpy()
        assert np.array_equal(g[mask].view(np.uint8), want[mask].view(np.uint8)), f"a poisoned {what} byte changed"


# ---- the reference sequence: q_to_fp16_kv -> attn_decode.cu -> fp16_to_q_kv ---------------------------------------------------

SENTINEL = 0x7BCD          # an fp16 bit pattern (~6.4e4) no conversion produces from these inputs


@pytest.mark.parametrize("wbits,hd", FMTS)
def test_reference_sequence_past_length(wbits, hd):
    from exllamav2_b200 import ext
    from exllamav2_b200.model import _lib
    KVH = 512 // hd                                   # a 512-value row: no widening to 512-value blocks
    H, q_len = 2 * KVH, 3
    seqlens = [0, 1, 255, 256, 257, 509]
    B, pps = len(seqlens), 2
    kb, vb = ar.widths(wbits)
    rng = np.random.default_rng(seed_of("ref", wbits, hd))
    pages_total = B * pps + 1
    bt = rng.permutation(pages_total)[:B * pps].reshape(B, pps).astype(np.int32)
    shp = (pages_total, PAGE, KVH)
    kq = rng.integers(0, 256, size=shp + (hd * kb // 8,), dtype=np.uint8)
    vq = rng.integers(0, 256, size=shp + (hd * vb // 8,), dtype=np.uint8)
    ks = (rng.uniform(0.05, 0.15, size=shp + (hd // 32,)) / (16 if kb == 8 else 1)).astype(np.float16)
    vs = (rng.uniform(0.02, 0.3, size=shp + (hd // 32,)) / (16 if vb == 8 else 1)).astype(np.float16)
    mask = poison_cache(rng, kq, ks, vq, vs, bt, seqlens, kb, vb)
    t = rg.t
    gk, gks, gv, gvs, sl, gbt = t(kq), t(ks), t(vq), t(vs), t(np.array(seqlens, np.int32)), t(bt)
    # 1. q_to_fp16_kv writes the live rows [0, seqlen) of each sequence into the temp, and nothing else
    tk = torch.full(shp + (hd,), SENTINEL, dtype=torch.int16, device=DEV).view(torch.half)
    tv = tk.clone()
    ext.q_to_fp16_kv(gk, tk, gks, gv, tv, gvs, B, 0, 0, PAGE, sl, gbt, wbits)
    torch.cuda.synchronize()
    live = ~mask
    for got, q_, s_, bits, what in ((tk, kq, ks, kb, "K"), (tv, vq, vs, vb, "V")):
        g = got.cpu().numpy()
        assert (g[mask].view(np.uint16) == SENTINEL).all(), f"q_to_fp16_kv wrote a {what} temp row past a length"
        want = kv_q68.kv_unpack(q_[live], s_[live], bits)
        assert np.allclose(g[live].astype(np.float64), want.astype(np.float64), rtol=2e-3, atol=1e-3), what
    # 2. attention over the temp, with fp16 rows past every length at up to +-2^12
    for tmp in (tk, tv):
        pz = torch.from_numpy(rng.uniform(-4096, 4096, size=(int(mask.sum()), KVH, hd)).astype(np.float16)).to(DEV)
        tmp[tuple(torch.from_numpy(a).to(DEV) for a in np.nonzero(mask))] = pz
    q = rng.normal(0, 4, size=(B, q_len, H, hd)).astype(np.float16)
    kn = rng.normal(0, 1, size=(B, q_len, KVH, hd)).astype(np.float16)
    vn = rng.normal(0, 1, size=(B, q_len, KVH, hd)).astype(np.float16)
    out = torch.zeros((B, q_len, H, hd), dtype=torch.half, device=DEV)
    kr = [tk.cpu().numpy()[bt[b][np.arange(s) // PAGE], np.arange(s) % PAGE].astype(np.float64) for b, s in enumerate(seqlens)]
    vr = [tv.cpu().numpy()[bt[b][np.arange(s) // PAGE], np.arange(s) % PAGE].astype(np.float64) for b, s in enumerate(seqlens)]
    gq, gkn, gvn = t(q), t(kn), t(vn)
    rc = _lib.exl2b_paged_attn_decode(gq.data_ptr(), gkn.data_ptr(), gvn.data_ptr(), tk.data_ptr(), tv.data_ptr(), sl.data_ptr(),
                                      gbt.data_ptr(), out.data_ptr(), B, q_len, H, KVH, hd, PAGE, pps, 1.0 / math.sqrt(hd),
                                      torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    truth = ar.attention_truth(q, kn, vn, kr, vr, seqlens, 1.0 / math.sqrt(hd))
    rg.compare(out.cpu().numpy(), truth, ("past_length", "attn_decode", wbits, hd))
    # 3. fp16_to_q_kv packs [seqlen, seqlen + q_len) of the temp (the new rows attn_decode.cu stored there), nothing else
    new = np.zeros(mask.shape, dtype=bool)
    for b, s in enumerate(seqlens):
        p = np.arange(s, s + q_len)
        new[bt[b][p // PAGE], p % PAGE] = True
    ext.fp16_to_q_kv(tk, gk, gks, tv, gv, gvs, B, 0, q_len, PAGE, sl, gbt, wbits)
    torch.cuda.synchronize()
    for got, want, what in ((gk, kq, "k"), (gks, ks, "k scales"), (gv, vq, "v"), (gvs, vs, "v scales")):
        g = got.cpu().numpy()
        assert np.array_equal(g[~new].view(np.uint8), want[~new].view(np.uint8)), f"fp16_to_q_kv wrote a {what} byte outside the new rows"
    for got_q, got_s, src, bits in ((gk, gks, kn, kb), (gv, gvs, vn, vb)):       # ... and those from the new rows
        gq_, gs_ = got_q.cpu().numpy(), got_s.cpu().numpy()
        for b, s in enumerate(seqlens):
            p = np.arange(s, s + q_len)
            rows = kv_q68.kv_unpack(gq_[bt[b][p // PAGE], p % PAGE], gs_[bt[b][p // PAGE], p % PAGE], bits).astype(np.float64)
            want = src[b].astype(np.float64)
            err = np.linalg.norm((rows - want).reshape(q_len, -1), axis=1) / np.linalg.norm(want.reshape(q_len, -1), axis=1)
            assert err.max() < 0.2, (b, err)
