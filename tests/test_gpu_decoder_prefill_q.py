"""ExLlamaV2Decoder.prefill_rows(ids, cache_attn=True) -- prompt attention straight over the quantised cache
(csrc/attn_prefill.cu) -- against the fp64 decoder truth (tests/decoder_truth.py), call by call, teacher-forced on the cache
bytes the decoder stored.

  P5  prefill_rows(cache_attn=True): gemm_big / wgmma blocks + paged_attn_prefill_q per layer; bound = P3's
Calls (B, T): (1, 40); (2, 10) then (2, 24) (past > 0); (1, 252) then decode steps across position 256 (the second page).
Each call asserts the branch: paged_attn_prefill_q once per layer, no q_to_fp16_kv / fp16_to_q_kv / _sdpa_prefill /
exl2b_paged_attn_decode.  Also: layer 0's appended cache bytes equal those of the default prefill_rows on the same prompt (its
inputs are identical there), and the whole call captured in a CUDA graph replays eager's bits."""
import numpy as np
import pytest
import torch

import decoder_truth as dt
from test_gpu_decoder_truth import DEV, SEED, _decoder, _ids, _truth_model

pytestmark = pytest.mark.gpu

MODELS = ["small", "tiny", "hd128", "gptq"]
CASES = [(m, b) for m in MODELS for b in (4, 6, 8)]
# (the GPTQ plan's 252-token prompt is checked in test_prompt_vs_fp64's models; its first decode step after it lands on an input
# whose fp16 floor is 4e-2, where the decode path -- not this prompt path -- measured 3.7x that floor, DESIGN.md §3.8)
LONG = [("small", 4), ("tiny", 6), ("hd128", 8)]


class PrefillSpy(dt.Spy):
    """dt.Spy plus the prompt attention entry point."""

    def __init__(self, monkeypatch):
        from exllamav2_b200 import ext
        super().__init__(monkeypatch)
        monkeypatch.setattr(ext, "paged_attn_prefill_q", self._wrap("paged_attn_prefill_q", ext.paged_attn_prefill_q))


def _check_branch(calls, L):
    names = dt.names_of(calls)
    assert len(dt.named(calls, "paged_attn_prefill_q")) == L
    assert len(dt.named(calls, "q_attn_forward_1")) == L and len(dt.named(calls, "q_mlp_forward_rows")) == L
    for n in ("q_to_fp16_kv", "fp16_to_q_kv", "_sdpa_prefill", "exl2b_paged_attn_decode", "paged_attn_decode_q4"):
        assert n not in names, f"cache_attn prefill reached {n}"


def _rows_call(dec, truth, ids, spy):
    pre, pos0 = dt.snapshot(dec), dec.pos
    spy.take()
    out = dec.prefill_rows(torch.from_numpy(ids).to(DEV), cache_attn=True).float().cpu().numpy()
    torch.cuda.synchronize()
    _check_branch(spy.take(), dec.cfg.num_layers)
    worst, floor, _ = dt.check_call(dec, truth, "P5", "rows", ids, out, pre, dt.snapshot(dec), pos0)
    print(f"TRUTH P5 {dec.cfg.name} Q{dec.cache.wbits} B={ids.shape[0]} T={ids.shape[1]} pos0={pos0}: rel-L2 {worst:.3e} "
          f"floor {floor:.3e}")


@pytest.fixture
def p5(monkeypatch):
    monkeypatch.setitem(dt.OUT_TOL, "P5", dt.OUT_TOL["P3"])
    return PrefillSpy(monkeypatch)


@pytest.mark.parametrize("model,bits", CASES, ids=[f"{m}-q{b}" for m, b in CASES])
def test_prompt_vs_fp64(model, bits, p5):
    for B, lens in ((1, [40]), (2, [10, 24])) + (((1, [252]),) if model == "gptq" and bits == 4 else ()):
        dec = _decoder(model, B, bits)
        try:
            truth = _truth_model(dec, SEED)
            for i, T in enumerate(lens):
                _rows_call(dec, truth, _ids(B, T, dec.cfg.vocab_size, 50 + i), p5)
        finally:
            dec.unload()


@pytest.mark.parametrize("model,bits", LONG, ids=[f"{m}-q{b}" for m, b in LONG])
def test_long_prompt_then_decode_across_a_page(model, bits, p5):
    from exllamav2_b200.model import PAGE_SIZE
    dec = _decoder(model, 1, bits)
    try:
        truth = _truth_model(dec, SEED)
        V = dec.cfg.vocab_size
        _rows_call(dec, truth, _ids(1, 252, V, 60), p5)
        for t in range(6):
            ids = _ids(1, 1, V, 70 + t)
            pre, pos0 = dt.snapshot(dec), dec.pos
            p5.take()
            out = dec.decode(torch.from_numpy(ids).to(DEV)).float().cpu().numpy()
            torch.cuda.synchronize()
            dt.check_branch("L", "decode", p5.take(), dec, dec.cfg.num_layers)
            dt.check_call(dec, truth, "L", "decode", ids, out, pre, dt.snapshot(dec), pos0)
        assert dec.pos > PAGE_SIZE
    finally:
        dec.unload()


@pytest.mark.parametrize("model,bits", [("small", 4), ("tiny", 8), ("hd128", 6), ("gptq", 4)])
def test_layer0_append_matches_default_path(model, bits):
    """Layer 0 sees the same inputs on both paths, so its appended bytes are the same; later layers differ by design (the prompt
    attention reads the cached values without the fp16 round trip)."""
    B, T = 2, 24
    ids = torch.from_numpy(_ids(B, T, 512, 80)).to(DEV)
    snaps = []
    for cache_attn in (False, True):
        dec = _decoder(model, B, bits)
        try:
            dec.prefill_rows(ids, cache_attn=cache_attn)
            torch.cuda.synchronize()
            snaps.append(dt.snapshot(dec))
        finally:
            dec.unload()
    for b in range(B):
        pg, r = dt.slots(snaps[0], b, 0, T)
        for key in ("k", "ks", "v", "vs"):
            a, c = snaps[0][key][0][pg, r], snaps[1][key][0][pg, r]
            assert np.array_equal(a.view(np.uint8), c.view(np.uint8)), f"seq {b}: layer 0 {key} differs from the default path"


@pytest.mark.parametrize("model,bits", [("tiny", 4), ("hd128", 8)])
def test_graph_capture_matches_eager(model, bits):
    dec = _decoder(model, 2, bits)
    try:
        c = dec.cache
        dec.prefill_rows(torch.from_numpy(_ids(2, 10, 512, 90)).to(DEV), cache_attn=True)      # past > 0, and the warm-up
        torch.cuda.synchronize()
        live = (*c.key_states, *c.key_scales, *c.value_states, *c.value_scales, c.cache_seqlens)
        state = [t.clone() for t in live]
        pos0 = dec.pos
        ids = torch.from_numpy(_ids(2, 30, 512, 91)).to(DEV)
        eager = dec.prefill_rows(ids, cache_attn=True).clone()
        torch.cuda.synchronize()
        eager_live = [t.clone() for t in live]
        for dst, src in zip(live, state):
            dst.copy_(src)
        dec.pos = pos0
        s = torch.cuda.Stream(DEV)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            out = dec.prefill_rows(ids, cache_attn=True)
        torch.cuda.synchronize()
        for dst, src in zip(live, state):          # (capture ran nothing; restore all the same)
            dst.copy_(src)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int16), eager.view(torch.int16)), "graph replay differs from the eager call"
        for a, b in zip(live, eager_live):
            assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), "graph replay stored different cache state"
    finally:
        dec.unload()
