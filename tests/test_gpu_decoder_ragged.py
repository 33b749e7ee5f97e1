"""Ragged batches through the whole decoder (exllamav2_b200/model.py ExLlamaV2Decoder) against the fp64 forward of
tests/decoder_truth.py: every sequence of a batch at its own length, and every cache row past a length poisoned.

A serving batch is ragged: sequences sit at different lengths, and one that just joined is at 0.  Each case builds that state
the way a server gets it: prefill_rows of one common prompt of the longest length, then cache_seqlens[b] set to each
sequence's own length (dec.pos, the host's mirror, to the longest), on a page table that is a random permutation of all
pages.  Every cache row at or past a sequence's length, in every layer, K and V, is then overwritten with random codes at a
scale where each dequantised element reaches ~2^12 (decoder_truth.poison_past): in every head about half of those rows score
far above any live row, so a launch that attends, sums or reads one of them moves the output by O(10^3).

Per call: the checks of decoder_truth.check_call with per-sequence starts (output per sequence within the §3.6 bound of its
schedule, past bytes unchanged, appended rows, seqlens advanced per sequence), every poisoned byte unchanged except the slot
the call appended into, the host branch (Spy / check_branch), and for every fused attention launch the regime the plan
restatement (tests/attn_regimes.py, tests/attn_long_plan.py) predicts for these lengths.  The truth of each sequence reads its
past from the decoder's own cache bytes, [0, its start): teacher forcing, so how accurate the prompt was does not matter.

  D5        chained, B = 3 and B = 8 (a full 8-row wgmma pass whose fused RoPE reads past_lens per row)
  D5-split  chained, B = 3, capacity 2048, lengths 1700 / 0 / 257: split-KV with a different chunk count per sequence
  D5-ring   chained, B = 3, hd 128, capacity 16 384, one sequence past 8192: the ring tail under split-KV
  D5-graph  as D5, captured: graph replay gives the eager step's bits on the ragged state, then the replayed steps are checked
  D6        un-chained fused, B = 9 and B = 16: two wgmma passes (the second at row 8), then the stand-alone rope_kernel
  D6-dense  ungrouped GPTQ (the wgmma kernel cannot stage it), B = 3: gemm_big + rope_launch at few rows
  D4        the reference sequence, B = 3: q_to_fp16_kv -> attn_decode.cu -> fp16_to_q_kv with per-sequence lengths
  P2        prefill(ids, 8) of 11 tokens onto ragged pasts, B = 3: 24 rows, then 9; appends crossing a page end in one sequence
  P3        prefill_rows onto ragged pasts: the fp16 temp + flash-attn where installed, the same with torch SDPA forced
            (_sdpa_prefill's per-sequence n0), and cache_attn=True (attn_prefill.cu)
Lengths across each schedule's cases include 0, 1, 255, 256, 257 and one sequence that ends the call at the capacity.
"""
import dataclasses

import numpy as np
import pytest
import torch

import attn_long_plan as alp
import attn_regimes as ar
import decoder_truth as dt
import test_gpu_decoder_prefill_q as tq
import test_gpu_decoder_truth as tt

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED = tt.SEED
MEASURED = {}


def _decoder(model, B, bits, cap, fused_attn=True, chained=True):
    from exllamav2_b200.model import ExLlamaV2Decoder
    cfg = tt._cfg(model)
    cfg = dataclasses.replace(cfg, max_seq_len=max(cfg.max_seq_len, cap))
    dec = ExLlamaV2Decoder(cfg, device=DEV, seed=SEED, batch_size=B, cache_len=cap, cache_bits=bits)
    dec.fused_attn, dec.chained = fused_attn, chained
    bt = dec.cache.block_table
    perm = torch.randperm(bt.numel(), generator=torch.Generator().manual_seed(2000 + B * 10 + bits)).to(torch.int32)
    if torch.equal(perm, torch.arange(bt.numel(), dtype=torch.int32)):
        perm = perm.roll(1)
    bt.copy_(perm.view(bt.shape).to(bt.device))
    return dec


def _ragged(dec, lens, rng):
    """prefill_rows of one common prompt of max(lens) tokens, then each sequence cut to its own length and everything past
    it poisoned.  Returns the poison (decoder_truth.poison_past)."""
    B, V = dec.batch_size, dec.cfg.vocab_size
    n = max(lens)
    prompt = np.repeat(rng.integers(0, V, size=(1, n)), B, axis=0).astype(np.int64)
    dec.prefill_rows(torch.from_numpy(prompt).to(DEV))
    torch.cuda.synchronize()
    dec.cache.cache_seqlens.copy_(torch.tensor(lens, dtype=torch.int32, device=DEV))
    dec.pos = max(lens)
    return dt.poison_past(dec, lens, rng)


def _regimes(calls, dec, starts):
    """The union of the branches the plan restatement gives the call's fused decode attention launches, each at the lengths
    it ran at: a prompt of several chunks advances the lengths by the chunk's q_len after every layer's launch."""
    L = dec.cfg.num_layers
    got, sl = set(), np.asarray(starts)
    for i, (a, kw) in enumerate(dt.named(calls, "paged_attn_decode_q4")):
        B, q_len, H, hd = a[0].shape
        max_ctx = a[3].shape[1] * a[8].shape[1]
        p = ar.plan(dec.cache.wbits, hd, H, B, q_len, max_ctx, sl.tolist())
        got |= ar.branches(p, q_len, H, B)
        if alp.long_plan(dec.cache.wbits, hd, H, B, q_len, max_ctx)["passes"]:
            got.add("passes")
        if q_len == 1 and any(c["ntail"] == 0 and c["c_hi"] - c["p_lo"] <= c["n_st"] for c in p["ctas"]):
            got.add("short")
        if i % L == L - 1:
            sl = sl + q_len
    return got


def _call(dec, truth, sched, kind, ids, spy, poison, tag, expect=None, branch_kind=None, **kw):
    pre = dt.snapshot(dec)
    starts = pre["seqlens"].astype(np.int64)
    spy.take()
    x = torch.from_numpy(ids).to(DEV)
    if kind == "decode":
        out = dec.decode(x)
    elif kind == "prefill":
        out = dec.prefill(x, 8)
    else:
        out = dec.prefill_rows(x, **kw)
    out = out.float().cpu().numpy()
    torch.cuda.synchronize()
    calls = spy.take()
    if dec.graph is None:
        dt.check_branch(sched, branch_kind or kind, calls, dec, dec.cfg.num_layers)
        got = _regimes(calls, dec, starts)
        assert expect is None or got == expect, (tag, expect, got)
    worst, floor, floored = dt.check_call(dec, truth, sched, kind, ids, out, pre, dt.snapshot(dec), starts, poison=poison)
    MEASURED[tag] = max(MEASURED.get(tag, 0.0), worst)
    print(f"TRUTH ragged {tag} {kind} starts {starts.tolist()}: out rel-L2 {worst:.3e} floor {floor:.3e} floored {floored}")
    return worst


# name: (schedule, model, Q, capacity, lens (B = len(lens)), fused_attn, chained, the branches the plan gives the step's
# attention launches (attn_regimes.branches, plus "short": a CTA takes the warp-local pass, "passes": attn_q4_passes_kernel))
G, S, M = {"global", "short"}, {"short"}, {"merge", "merge_batch"}
DECODE = {
    "D5-small-b3": ("D5", "small", 4, 512, [0, 256, 509], True, True, S),
    "D5-tiny-b8": ("D5", "tiny", 6, 512, [0, 1, 255, 256, 257, 100, 509, 30], True, True, G),
    "D5-hd128-b3": ("D5", "hd128", 8, 512, [1, 255, 257], True, True, G),
    "D5-split": ("D5", "small", 6, 2048, [1700, 0, 257], True, True, G | M),
    "D5-ring": ("D5", "hd128", 4, 16384, [8300, 1, 256], True, True, S | M | {"ring"}),
    "D6-small-b9": ("D6", "small", 4, 512, [0, 1, 255, 256, 257, 303, 509, 17, 128], True, True, S),
    "D6-tiny-b16": ("D6", "tiny", 8, 512, [0, 1, 255, 256, 257, 509, 2, 3, 60, 61, 127, 128, 129, 300, 400, 500], True, True, G),
    "D6-hd128-b9": ("D6", "hd128", 6, 512, [509, 0, 1, 255, 256, 257, 40, 300, 100], True, True, G),
    "D6-dense": ("D5", "gptq-nogroup", 4, 512, [257, 0, 509], True, True, S),
    "D4-small": ("D4", "small", 6, 512, [256, 0, 509], False, False, set()),
    "D4-hd128": ("D4", "hd128", 4, 512, [1, 257, 255], False, False, set()),
}


@pytest.mark.parametrize("name", list(DECODE))
def test_ragged_decode(name, monkeypatch, request):
    sched, model, bits, cap, lens, fused, chained, expect = DECODE[name]
    if tt._in_child(request, True):
        return
    B = len(lens)
    dec = _decoder(model, B, bits, cap, fused, chained)
    try:
        assert max(lens) + 3 <= cap
        if name == "D6-dense":      # a matrix the wgmma kernel cannot stage: Q|K|V take gemm_big + rope_launch (blocks.cu)
            assert not dec.tc_staged
        truth = tt._truth_model(dec, SEED)
        rng = np.random.default_rng(sum(map(ord, name)))
        poison = _ragged(dec, lens, rng)
        spy = dt.Spy(monkeypatch)
        for t in range(3):
            _call(dec, truth, sched, "decode", tt._ids(B, 1, dec.cfg.vocab_size, 10 + t), spy, poison, name, expect)
        assert dec.pos == max(lens) + 3
    finally:
        dec.unload()


def test_ragged_decode_graph(monkeypatch, request):
    """D5 captured on a ragged, poisoned state: each replayed step gives the eager step's bits, then is checked itself."""
    if tt._in_child(request, True):
        return
    lens = [257, 0, 1]
    dec = _decoder("small", 3, 8, 512)
    try:
        truth = tt._truth_model(dec, SEED)
        poison = _ragged(dec, lens, np.random.default_rng(11))
        spy = dt.Spy(monkeypatch)
        dec.capture()
        for t in range(3):
            ids = tt._ids(3, 1, dec.cfg.vocab_size, 30 + t)
            spy.take()
            dt.graph_matches_eager(dec, ids, lambda: dt.check_branch("D5", "decode", spy.take(), dec, dec.cfg.num_layers))
            _call(dec, truth, "D5", "decode", ids, spy, poison, "D5-graph")
    finally:
        dec.unload()


# name: (schedule, model, Q, capacity, lens, kind, T, prefill_rows keyword arguments, the branches of the prompt's fused decode
# attention launches (prefill_rows has none), those of the decode step after it)
PROMPT = {
    "P2-small": ("P2", "small", 4, 512, [250, 0, 100], "prefill", 11, {}, set(), S),
    "P2-hd128": ("P2", "hd128", 8, 512, [1, 245, 256], "prefill", 11, {}, {"global"}, G),
    "P3-small": ("P3", "small", 4, 512, [257, 0], "rows", 10, {}, set(), S),
    "P3-hd128": ("P3", "hd128", 6, 512, [1, 255, 256], "rows", 12, {}, set(), S),
    "P3-small-sdpa": ("P3", "small", 4, 512, [257, 0], "rows", 10, {}, set(), S),
    "P3-hd128-sdpa": ("P3", "hd128", 6, 512, [1, 255, 256], "rows", 12, {}, set(), S),
    "P3-q-small": ("P3", "small", 8, 512, [0, 256, 300], "rows", 10, dict(cache_attn=True), set(), G),
    "P3-q-hd128": ("P3", "hd128", 4, 512, [255, 1], "rows", 9, dict(cache_attn=True), set(), S),
}


@pytest.mark.parametrize("name", list(PROMPT))
def test_ragged_prompt(name, monkeypatch, request):
    from exllamav2_b200 import model as model_mod
    sched, model, bits, cap, lens, kind, T, kw, expect, expect_decode = PROMPT[name]
    if name.endswith("-sdpa"):          # prompt attention by torch SDPA (_sdpa_prefill) even where flash-attn is installed
        monkeypatch.setattr(model_mod, "_FA", [True, None])
    if tt._in_child(request, True):
        return
    B = len(lens)
    dec = _decoder(model, B, bits, cap)
    try:
        truth = tt._truth_model(dec, SEED)
        poison = _ragged(dec, lens, np.random.default_rng(sum(map(ord, name))))
        spy = tq.PrefillSpy(monkeypatch)
        _call(dec, truth, sched, kind, tt._ids(B, T, dec.cfg.vocab_size, 40), spy, poison, name, expect,
              branch_kind="rows_q" if kw.get("cache_attn") else None, **kw)
        # then a decode step on the state the prompt left: every sequence one past its ragged end
        _call(dec, truth, "D5", "decode", tt._ids(B, 1, dec.cfg.vocab_size, 41), spy, poison, name + "-decode", expect_decode)
    finally:
        dec.unload()


def test_replay_fused_step_matches_decode(monkeypatch, request):
    """decoder_truth.replay_fused_step issues the D6 step's launches one at a time: on a ragged, poisoned B = 9 state it gives
    decode()'s logits and cache bytes bit for bit, and every launch is within its own bound (decoder_truth.LAUNCH_TOL)."""
    if tt._in_child(request, True):
        return
    lens = [0, 1, 255, 256, 257, 303, 509, 17, 128]
    dec = _decoder("small", 9, 6, 512)
    try:
        _ragged(dec, lens, np.random.default_rng(5))
        c = dec.cache
        live = (*c.key_states, *c.key_scales, *c.value_states, *c.value_scales, c.cache_seqlens)
        state = [t.clone() for t in live]
        ids = tt._ids(9, 1, dec.cfg.vocab_size, 60)
        want = dec.decode(torch.from_numpy(ids).to(DEV)).clone()
        want_live = [t.clone() for t in live]
        for d, s in zip(live, state):
            d.copy_(s)
        dec.pos -= 1
        errs = dt.replay_fused_step(dec, ids)
        assert torch.equal(dec.logits.view(torch.int16), want.view(torch.int16)), "the replay differs from decode()"
        for a, b in zip(live, want_live):
            assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), "the replay stored different cache state"
        assert dec.pos == max(lens) + 1
        for (launch, li), e in errs.items():
            print(f"REPLAY {launch} layer {li}: worst rel-L2 {e.max():.3e}")
            assert e.max() <= dt.LAUNCH_TOL[launch], (launch, li, e)
    finally:
        dec.unload()


def test_report_worst():
    for k, v in sorted(MEASURED.items()):
        print(f"RAGGED worst {k}: {v:.3e}")
