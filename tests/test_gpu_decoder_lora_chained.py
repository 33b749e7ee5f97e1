"""Batch-1 decode with LoRA adapters on the chained step (include/exl2_b200.h "block forwards", csrc/lora.cu's one-row form).

- Zero-B adapters (B = 0) on all seven projections leave the chained step's logits byte-identical to the adapter-free chained
  step's, eager and graph-replayed, on the 7B preset and test-small: a wrong mirror index or an ordering hazard between a LoRA
  launch and its neighbours would show here.
- Launch counts on the 7B preset: 161 + 32 per adapted stage.
- The schedule, from the extension calls: chained at batch 1, the un-chained forms at batch 2 and 8.
- Against the fp64 forward with the adapters' terms (test_gpu_decoder_lora's LoraTruth), under D1's bound, on test-small and the
  hd-128 GQA model, Q4 / Q6 / Q8 caches, with adapters of rank 16 on all seven, 64 on q and v, and 13 on o and down; eager steps,
  then a captured graph whose replay equals the eager step.
- On the 7B preset, the chained adapted step against the un-chained adapted step.
- A chained call of two rows with an active adapter is refused."""

import numpy as np
import pytest
import torch

import decoder_truth as dt
from test_gpu_decoder_lora import _cfg, _check, _ids, _truth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ALL = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")


def _reset(dec):
    dec.graph = None
    dec.cache.cache_seqlens.zero_()
    dec.pos = 0


def _steps(dec, toks, graph):
    """decode toks [(1, 1) ids] from position 0, eager or replaying a graph captured at position 0; the logits of every step"""
    _reset(dec)
    if graph:
        dec.capture()
    return [dec.decode(t).clone() for t in toks]


@pytest.fixture(scope="module")
def dec7b():
    from exllamav2_b200.model import PRESETS, ExLlamaV2Decoder
    dec = ExLlamaV2Decoder(PRESETS["llama2-7b-4.0bpw"](), device=DEV, seed=0, cache_len=512)
    yield dec
    dec.unload()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def dec_small():
    from exllamav2_b200.model import PRESETS, ExLlamaV2Decoder
    dec = ExLlamaV2Decoder(PRESETS["test-small"](), device=DEV, seed=5, cache_len=512)
    yield dec
    dec.unload()


@pytest.mark.parametrize("model", ["7b", "small"])
def test_zero_b_is_byte_identical(model, request):
    dec = request.getfixturevalue("dec7b" if model == "7b" else "dec_small")
    V = dec.cfg.vocab_size
    toks = [torch.tensor([[int(t)]], device=DEV) for t in np.random.default_rng(7).integers(0, V, 5)]
    dec.set_loras([])
    plain = {g: _steps(dec, toks, g) for g in (False, True)}
    key = dec.load_lora(16, targets=ALL, scaling=0.0, seed=1)
    dec.set_loras([key])
    assert dec._chains(1)
    try:
        for g in (False, True):
            got = _steps(dec, toks, g)
            for s, (a, b) in enumerate(zip(got, plain[g])):
                assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"{model} {'graph' if g else 'eager'} step {s}"
        assert torch.equal(plain[True][-1].view(torch.int16), plain[False][-1].view(torch.int16))
    finally:
        _reset(dec)
        dec.unload_lora(key)


def test_launch_counts_7b(dec7b):
    from exllamav2_b200 import ext
    dec = dec7b
    ids = torch.tensor([[17]], device=DEV)

    def count():
        _reset(dec)
        torch.cuda.synchronize()
        n0 = ext.launch_count()
        dec.decode(ids)
        torch.cuda.synchronize()
        return ext.launch_count() - n0

    qv = dec.load_lora(16, targets=("q_proj", "v_proj"), seed=1)
    full = dec.load_lora(16, targets=ALL, seed=2)
    try:
        dec.set_loras([qv])
        assert count() == 161 + 32          # q|k|v adapted
        dec.set_loras([full])
        assert count() == 161 + 4 * 32      # q|k|v, o, gate|up, down
        dec.set_loras([qv, full])
        assert count() == 161 + 4 * 32      # one LoRA launch per adapted stage, whatever the adapters
        dec.set_loras([])
        assert count() == 161
    finally:
        _reset(dec)
        dec.unload_lora(qv)
        dec.unload_lora(full)


@pytest.mark.parametrize("B", [1, 2, 8])
def test_schedule(B, monkeypatch):
    from exllamav2_b200 import ext
    from exllamav2_b200.model import ExLlamaV2Decoder
    dec = ExLlamaV2Decoder(_cfg("small"), device=DEV, seed=3, batch_size=B, cache_len=512)
    dec.set_loras([dec.load_lora(16, seed=1)])
    spy = dt.Spy(monkeypatch)
    for name in ("q_attn_forward_2_ex", "q_attn_forward_2"):
        monkeypatch.setattr(ext, name, spy._wrap(name, getattr(ext, name)))
    dec.decode(torch.from_numpy(_ids(B, 1, dec.cfg.vocab_size, 4)).to(DEV))
    torch.cuda.synchronize()
    calls = spy.take()
    L, ids = dec.cfg.num_layers, dec.lora_ids
    if B == 1:
        dt.check_branch("D1", "decode", calls, dec, L)
        assert [a[12] for a, _ in dt.named(calls, "q_attn_forward_1_ex")] == [ids] * L
        assert [a[7] for a, _ in dt.named(calls, "q_attn_forward_2_ex")] == [ids] * L
        assert [a[4] for a, _ in dt.named(calls, "q_mlp_forward_ex")] == [ids] * L
        assert not {"q_attn_forward_1", "q_attn_forward_2", "q_mlp_forward_"} & dt.names_of(calls)
    else:
        assert not {"q_attn_forward_1_ex", "q_attn_forward_2_ex", "q_mlp_forward_ex"} & dt.names_of(calls)
        assert [(a[2], a[3], a[11]) for a, _ in dt.named(calls, "q_attn_forward_1")] == [(B, 1, ids)] * L
        assert [a[5] for a, _ in dt.named(calls, "q_attn_forward_2")] == [ids] * L
        assert [a[2] for a, _ in dt.named(calls, "q_mlp_forward_")] == [ids] * L
        assert len(dt.named(calls, "paged_attn_decode_q4")) == L
        assert {"gemv_norm", "gemm_half_q_half_prepared", "gemm_half_q_half"} & dt.names_of(calls) == {"gemm_half_q_half"}
    dec.unload()


@pytest.mark.parametrize("bits", [4, 6, 8])
@pytest.mark.parametrize("model", ["small", "hd128"])
def test_decode_b1_vs_fp64(model, bits):
    from exllamav2_b200.model import ExLlamaV2Decoder
    dec = ExLlamaV2Decoder(_cfg(model), device=DEV, seed=3, batch_size=1, cache_len=512, cache_bits=bits)
    a = dec.load_lora(16, seed=1)                                                # every projection
    b = dec.load_lora(64, targets=("q_proj", "v_proj"), scaling=0.5, seed=2)
    c = dec.load_lora(13, targets=("o_proj", "down_proj"), seed=3)              # an odd rank
    dec.set_loras([a, b, c])
    assert dec._chains(1)
    truth = _truth(dec)
    V = dec.cfg.vocab_size
    _check(dec, truth, "P1", "prefill", _ids(1, 11, V, 1), lambda x: dec.prefill(x, 8))
    worst = 0.0
    for s in range(6):
        worst = max(worst, _check(dec, truth, "D1", "decode", _ids(1, 1, V, 10 + s), dec.decode))
    dec.capture()
    dt.graph_matches_eager(dec, _ids(1, 1, V, 20))
    for s in range(3):
        worst = max(worst, _check(dec, truth, "D1", "decode", _ids(1, 1, V, 30 + s), dec.decode))
    print(f"CHAINED LORA {model} Q{bits}: worst decode rel-L2 {worst:.3e} (bound {dt.OUT_TOL['D1']})")
    dec.unload()


@pytest.mark.parametrize("targets", [("q_proj", "v_proj"), ALL], ids=["qv", "all"])
def test_7b_chained_vs_unchained(dec7b, targets):
    from exl2_oracle import rel_l2
    dec = dec7b
    key = dec.load_lora(16, targets=targets, seed=4)
    dec.set_loras([key])
    toks = [torch.tensor([[int(t)]], device=DEV) for t in np.random.default_rng(8).integers(0, dec.cfg.vocab_size, 4)]
    try:
        chained = _steps(dec, toks, False)
        dec.chained = False
        unchained = _steps(dec, toks, False)
    finally:
        dec.chained = True
        _reset(dec)
        dec.unload_lora(key)
    errs = [rel_l2(a.float().cpu().numpy().astype(np.float64), b.float().cpu().numpy().astype(np.float64))
            for a, b in zip(chained, unchained)]
    print(f"7B {'+'.join(t[0] for t in targets)} rank 16: chained vs un-chained logits rel-L2 per step {['%.2e' % e for e in errs]}")
    assert max(errs) <= 5e-3


def test_two_rows_refused():
    from exllamav2_b200 import ext
    from exllamav2_b200.model import ExLlamaV2Decoder
    dec = ExLlamaV2Decoder(_cfg("small"), device=DEV, seed=3, batch_size=2, cache_len=512)
    dec.set_loras([dec.load_lora(16, seed=1)])
    L, ids, c = dec.layers[0], dec.lora_ids, dec.cache
    with pytest.raises(RuntimeError, match="above one row"):
        ext.q_attn_forward_1_ex(L.attn, dec.x, 2, 1, -1, c.cache_seqlens, dec.q, dec.k, dec.v, dec.sin, dec.cos, True, ids)
    with pytest.raises(RuntimeError, match="above one row"):
        ext.q_attn_forward_2_ex(L.attn, dec.x, dec.attn_out, 2, 1, True, L.chain_mlp, ids)
    with pytest.raises(RuntimeError, match="above one row"):
        ext.q_mlp_forward_ex(L.mlp, dec.x, True, dec.layers[1].chain_attn, ids)
    # without adapters the same chained call runs
    dec.x.zero_()
    ext.q_mlp_forward_ex(L.mlp, dec.x, False, dec.layers[1].chain_attn)
    torch.cuda.synchronize()
    dec.unload()
