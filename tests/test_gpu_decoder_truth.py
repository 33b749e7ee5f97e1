"""The whole decoder (exllamav2_b200/model.py ExLlamaV2Decoder) against an fp64 Llama forward (tests/decoder_truth.py), call by
call, teacher-forced on the K/V cache bytes the decoder itself stored.

Every decode and prompt schedule the decoder has is run here, on a page table that is a random permutation of all pages:

  D1  B = 1, chained, row_gemv (eager and graph replay)   i8 GEMV, RoPE inside attention, gemv_norm(prepared) head
  D2  B = 1, chained, EXL2B_GEMV=tc (child process)      one-row wgmma chain, gemm_half_q_half_prepared head
  D3  B = 1, fused, not chained                           i8 GEMV + stand-alone RoPE, q_mlp_forward_, rms_norm + gemm head
  D4  B = 1, reference sequence                           q_to_fp16_kv -> fp16 attention -> fp16_to_q_kv
  D5  B = 3, chained                                      batched chain, prepared head
  D6  B = 12                                              non-chained fused branch, 12-row wgmma, rms_norm + gemm head
  P1  prefill chunk 8, B = 1, T = 11                      chained q_len 8, then 3
  P2  prefill chunk 8, B = 3, T = 11                      24-row chunk through gemm_big + fused attention q_len 8, then 9 rows
  P3  prefill_rows (B, T) = (1, 40), (2, 10 + 24), (1, 12) gemm_big + prompt attention on the fp16 temp; past > 0; <= 16 rows
      (-sdpa: torch SDPA forced even where flash-attn is installed)
  P4  prefill, reference sequence                         fp16 attention for chunks
  L   prefill_rows of 252 tokens, then D1 steps across position 256 (the second page)

Models: test-small (MHA, hd 64, 512-wide kv row), test-tiny (GQA, hd 64, 128-wide kv row: fused schedules only -- the reference
sequence re-quantises neighbouring tokens there, a documented divergence), a 2-layer hd-128 GQA model and, on test-small's
dimensions, a GPTQ g128 act-order plan, an all-8-bit g128 EXL2 plan (groups exactly at the wgmma kernel's 4 KB stage) and an
ungrouped act-order GPTQ plan (groups it cannot stage: above one row its steps take the fused, un-chained branch); K/V cache
Q4 / Q6 / Q8.

Per call: (1) logits (decode) or the returned hidden state (prompt) per sequence vs the fp64 truth, rel-L2 below a measured
bound per schedule (DESIGN.md §3.6), scaled up only on inputs whose fp16 floor is atypically large (decoder_truth.FLOOR_TYPICAL);
(2) cache bytes at positions written before the call unchanged, and each appended row, dequantised, no further from the truth
row than 1.1x the format's own quantisation error of that row plus a small slack; (3) cache_seqlens and dec.pos advanced by
exactly the tokens fed; (4) D1: graph replay produces eager's bits.  Each call also asserts the host branch it took, from the
extension entry points it reached (Spy), and the decoder's RoPE tables are pinned against exact sin / cos."""
import math

import numpy as np
import pytest
import torch

import decoder_truth as dt
import exl2_oracle as oracle

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED = 3
CACHE_LEN = 512         # 2 pages per sequence

OUT_TOL = dt.OUT_TOL     # per-schedule output bounds and the fp16-floor / K/V-row rules: tests/decoder_truth.py


# ---- models -------------------------------------------------------------------------------------------------------------

def _cfg(model):
    from exllamav2_b200.model import PRESETS, LlamaConfig, QuantPlan
    if model == "small":
        return PRESETS["test-small"]()
    if model == "tiny":
        return PRESETS["test-tiny"]()
    if model == "hd128":        # GQA, hd 128: kv row 4 x 128 = 512 values, so the reference sequence is valid too
        return LlamaConfig("test-hd128-gqa", 1024, 2816, 8, 4, 128, 2, 1024, max_seq_len=512, plan=PRESETS["test-small"]().plan)
    if model == "gptq":
        return LlamaConfig("test-small-gptq", 512, 1408, 8, 8, 64, 2, 512, max_seq_len=512,
                           plan=QuantPlan(attn=("gptq", 128, True), mlp=[("gptq", 128, True)], head=((6,), (1.0,), 128)))
    if model == "exl2-8bpw":     # every linear 8-bit g128, head included: groups exactly at the wgmma kernel's 4 KB stage
        b8 = ((8,), (1.0,), 128)
        return LlamaConfig("test-small-8bpw", 512, 1408, 8, 8, 64, 2, 512, max_seq_len=512, plan=QuantPlan(attn=b8, mlp=[b8], head=b8))
    if model == "gptq-nogroup":  # ungrouped act-order GPTQ (group_size -1): groups the wgmma kernel cannot stage
        return LlamaConfig("test-small-gptq-nogroup", 512, 1408, 8, 8, 64, 2, 512, max_seq_len=512,
                           plan=QuantPlan(attn=("gptq", -1, True), mlp=[("gptq", -1, True)], head=((6,), (1.0,), 128)))
    raise KeyError(model)


_ORACLE_W = {}


def _oracle_weights(cfg, seed):
    """fp16 W[K, N] of every linear in the decoder's order (per layer q, k, v, o, gate, up, down; then the head), regenerated
    from the decoder's seed schedule and reconstructed by the numpy oracle.  Fresh tensors: make_q_matrix scales q_scale_max
    in place, so the decoder's own q_tensors are not the checkpoint any more."""
    from exllamav2_b200 import synthetic
    key = (cfg.name, seed)
    if key in _ORACLE_W:
        return _ORACLE_W[key]
    H, KVH, hd, hid, inter = cfg.num_heads, cfg.num_kv_heads, cfg.head_dim, cfg.hidden_size, cfg.intermediate_size
    out = []

    def one(K, N, plan, s, perm_seed=None):
        w = synthetic.random_linear(K, N, plan, device=DEV, seed=s, weight_std=1.0 / math.sqrt(K), perm_seed=perm_seed)
        w = {k: v.cpu().numpy() for k, v in w.items()}
        out.append(oracle.gptq_reconstruct(w) if plan[0] == "gptq" else oracle.exl2_reconstruct(w))

    s = seed * 100003
    for li in range(cfg.num_layers):
        mp = cfg.plan.mlp[li % len(cfg.plan.mlp)]
        one(hid, H * hd, cfg.plan.attn, s + 1, s + 1)
        one(hid, KVH * hd, cfg.plan.attn, s + 2, s + 1)
        one(hid, KVH * hd, cfg.plan.attn, s + 3, s + 1)
        one(H * hd, hid, cfg.plan.attn, s + 4)
        one(hid, inter, mp, s + 5, s + 5)
        one(hid, inter, mp, s + 6, s + 5)
        one(inter, hid, mp, s + 7)
        s += 16
    one(hid, cfg.vocab_size, cfg.plan.head, s + 9)
    _ORACLE_W[key] = out
    return out


def _truth_model(dec, seed):
    cfg = dec.cfg
    W = _oracle_weights(cfg, seed)
    assert len(W) == len(dec.linears)
    for i, (lin, w) in enumerate(zip(dec.linears, W)):     # guards the seed schedule: the truth runs the decoder's weights
        got = lin.get_weight_tensor_dq().cpu().numpy()
        assert np.array_equal(got.view(np.uint16), w.view(np.uint16)), f"linear {i}: oracle reconstruction differs"
    f64 = [w.astype(np.float64) for w in W]
    # the truth rotates with the decoder's own tables, so they are pinned here against the exact angles: a table that is off by a
    # position rotates every query and key alike and leaves every score unchanged (RoPE is relative), invisible downstream
    n, hd = dec.sin.shape[0], cfg.head_dim
    ang = np.arange(n)[:, None] * (1.0 / cfg.rope_theta ** (np.arange(0, hd, 2) / hd))[None, :]
    ang = np.concatenate([ang, ang], axis=-1)
    # (the tables are built in fp32 as the reference builds them: an angle p x f is off by up to ~p x 2^-23 before the fp16
    # rounding, which matters only for tables much longer than these models' 512 positions)
    for tab, want in ((dec.sin, np.sin(ang)), (dec.cos, np.cos(ang))):
        assert np.abs(tab.float().cpu().numpy() - want).max() <= 1e-3 + n * 2.0 ** -23, \
            "RoPE table differs from sin / cos of position x frequency"

    def h(t):
        return t.float().cpu().numpy().astype(np.float64)

    layers = []
    for li, L in enumerate(dec.layers):
        wq, wk, wv, wo, wg, wu, wd = f64[7 * li:7 * li + 7]
        layers.append(dt.TruthLayer(h(L.input_norm), h(L.post_norm), wq, wk, wv, wo, wg, wu, wd))
    return dt.TruthModel(layers, h(dec.final_norm), f64[-1], h(dec.embed), h(dec.sin), h(dec.cos), cfg.num_heads,
                         cfg.num_kv_heads, cfg.head_dim, cfg.norm_eps)


def _decoder(model, B, bits, fused_attn=True, chained=True, row_gemv=True):
    from exllamav2_b200.model import ExLlamaV2Decoder
    dec = ExLlamaV2Decoder(_cfg(model), device=DEV, seed=SEED, batch_size=B, cache_len=CACHE_LEN, cache_bits=bits)
    dec.fused_attn, dec.chained = fused_attn, chained
    assert dec.row_gemv == row_gemv       # the library's single-row path (EXL2B_GEMV at load), see _in_child
    # a non-identity page table: every sequence's pages are scattered over the pool
    bt = dec.cache.block_table
    perm = torch.randperm(bt.numel(), generator=torch.Generator().manual_seed(1000 + B * 10 + bits)).to(torch.int32)
    if torch.equal(perm, torch.arange(bt.numel(), dtype=torch.int32)):
        perm = perm.roll(1)
    bt.copy_(perm.view(bt.shape).to(bt.device))
    return dec


def _in_child(request, row_gemv):
    """The single-row path is chosen by the library once, at load (EXL2B_GEMV=tc: wgmma; default: integer GEMV).  A case that
    needs the other path than this process has runs in a child process that loads the library with it.  True if it ran
    there (and passed)."""
    import os
    import subprocess
    import sys
    from exllamav2_b200 import ext
    if ext.row_gemv_i8() == row_gemv:
        return False
    env = dict(os.environ)
    env.pop("EXL2B_GEMV", None)
    if not row_gemv:
        env["EXL2B_GEMV"] = "tc"
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-s", "-p", "no:cacheprovider", f"{request.path}::{request.node.name}"],
                       env=env, capture_output=True, text=True)
    print(r.stdout[-4000:])
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    return True


# ---- one call, checked ----------------------------------------------------------------------------------------------------

def _call(dec, truth, sched, kind, ids, spy, chunk=8):
    """Run one decoder call over ids [B, T] and check it against the truth.  Returns the worst output rel-L2."""
    cfg, bits = dec.cfg, dec.cache.wbits
    B, T = ids.shape
    L = cfg.num_layers
    pre = dt.snapshot(dec)
    pos0 = dec.pos
    assert (pre["seqlens"] == pos0).all()
    spy.take()
    ids_d = torch.from_numpy(ids).to(DEV)
    if kind == "decode":
        out = dec.decode(ids_d).float().cpu().numpy()
    elif kind == "prefill":
        out = dec.prefill(ids_d, chunk).float().cpu().numpy()
    else:
        out = dec.prefill_rows(ids_d).float().cpu().numpy()
    torch.cuda.synchronize()
    calls = spy.take()
    if dec.graph is None:           # (a replayed step reaches no entry point: its eager twin is checked instead)
        dt.check_branch(sched, kind, calls, dec, L)
    worst, worst_floor, floored = dt.check_call(dec, truth, sched, kind, ids, out, pre, dt.snapshot(dec), pos0, chunk)
    print(f"TRUTH {sched} {cfg.name} Q{bits} {kind} B={B} T={T} pos0={pos0}: out rel-L2 {worst:.3e} floor {worst_floor:.3e} "
          f"floored {floored}")
    return worst


def _ids(B, T, vocab, seed):
    return np.random.default_rng(seed).integers(0, vocab, size=(B, T)).astype(np.int64)


# ---- decode schedules -----------------------------------------------------------------------------------------------------

DECODE_FLAGS = {    # B, fused_attn, chained, row_gemv
    "D1": (1, True, True, True),
    "D2": (1, True, True, False),
    "D3": (1, True, False, True),
    "D4": (1, False, False, True),
    "D5": (3, True, True, True),
    "D6": (12, True, True, True),
}

DECODE_CASES = [
    ("D1", "small", 4), ("D1", "small", 6), ("D1", "small", 8), ("D1", "tiny", 4), ("D1", "hd128", 4), ("D1", "hd128", 8),
    ("D1", "gptq", 4),
    ("D2", "small", 4), ("D2", "tiny", 6), ("D2", "hd128", 6), ("D2", "gptq", 8),
    ("D3", "small", 4), ("D3", "tiny", 8), ("D3", "hd128", 4), ("D3", "gptq", 6),
    ("D4", "small", 4), ("D4", "small", 6), ("D4", "small", 8), ("D4", "hd128", 4), ("D4", "gptq", 4),
    ("D5", "small", 4), ("D5", "tiny", 4), ("D5", "hd128", 8), ("D5", "gptq", 4),
    ("D6", "small", 4), ("D6", "tiny", 6), ("D6", "hd128", 4), ("D6", "gptq", 8),
    ("D1", "exl2-8bpw", 4), ("D1", "gptq-nogroup", 8), ("D5", "exl2-8bpw", 6), ("D5", "gptq-nogroup", 4),
]


@pytest.mark.parametrize("sched,model,bits", DECODE_CASES, ids=[f"{s}-{m}-q{b}" for s, m, b in DECODE_CASES])
def test_decode_vs_fp64(sched, model, bits, monkeypatch, request):
    B, fused, chained, row_gemv = DECODE_FLAGS[sched]
    if _in_child(request, row_gemv):
        return
    dec = _decoder(model, B, bits, fused, chained, row_gemv)
    try:
        truth = _truth_model(dec, SEED)
        spy = dt.Spy(monkeypatch)
        V = dec.cfg.vocab_size
        _call(dec, truth, sched, "prefill", _ids(B, 9, V, 1), spy)
        graph = sched == "D1"
        if graph:
            dec.capture()
        for t in range(3):
            ids = _ids(B, 1, V, 10 + t)
            if graph:
                _graph_matches_eager(dec, ids, spy)
            _call(dec, truth, sched, "decode", ids, spy)
    finally:
        dec.unload()


def _graph_matches_eager(dec, ids, spy):
    """(4) graph replay produces eager's bits (decoder_truth.graph_matches_eager), the eager step on the D1 branch."""
    spy.take()
    dt.graph_matches_eager(dec, ids, lambda: dt.check_branch("D1", "decode", spy.take(), dec, dec.cfg.num_layers))


# ---- prompt schedules -----------------------------------------------------------------------------------------------------

PROMPT = {   # B, fused_attn, chained, row_gemv, kind, prompt lengths (one call each)
    "P1": (1, True, True, True, "prefill", [11]),
    "P2": (3, True, True, True, "prefill", [11]),
    "P3a": (1, True, True, True, "rows", [40]),
    "P3b": (2, True, True, True, "rows", [10, 24]),
    "P3c": (1, True, True, True, "rows", [12]),
    "P4": (1, False, False, True, "prefill", [11]),
}
SDPA = {"P3a-sdpa": "P3a", "P3b-sdpa": "P3b"}    # prompt attention by torch SDPA even where flash-attn is installed

PROMPT_CASES = [
    ("P1", "small", 4), ("P1", "small", 6), ("P1", "small", 8), ("P1", "tiny", 4), ("P1", "hd128", 6), ("P1", "gptq", 4),
    ("P2", "small", 4), ("P2", "tiny", 6), ("P2", "hd128", 4), ("P2", "gptq", 8),
    ("P3a", "small", 4), ("P3a", "small", 6), ("P3a", "small", 8), ("P3a", "hd128", 4), ("P3a", "gptq", 4),
    ("P3b", "small", 4), ("P3b", "hd128", 8), ("P3b", "gptq", 6),
    ("P3c", "small", 4), ("P3c", "small", 8), ("P3c", "hd128", 6),
    ("P3a-sdpa", "small", 4), ("P3a-sdpa", "hd128", 8), ("P3b-sdpa", "small", 6), ("P3b-sdpa", "gptq", 4),
    ("P4", "small", 4), ("P4", "small", 6), ("P4", "small", 8), ("P4", "hd128", 4), ("P4", "gptq", 4),
    ("P1", "exl2-8bpw", 4), ("P1", "gptq-nogroup", 6), ("P2", "exl2-8bpw", 8), ("P2", "gptq-nogroup", 4),
    ("P3a", "exl2-8bpw", 6), ("P3a", "gptq-nogroup", 4), ("P3b", "gptq-nogroup", 8), ("P3c", "exl2-8bpw", 4),
    ("P3c", "gptq-nogroup", 6),
]


@pytest.mark.parametrize("sched,model,bits", PROMPT_CASES, ids=[f"{s}-{m}-q{b}" for s, m, b in PROMPT_CASES])
def test_prompt_vs_fp64(sched, model, bits, monkeypatch, request):
    from exllamav2_b200 import model as model_mod
    if sched in SDPA:
        monkeypatch.setattr(model_mod, "_FA", [True, None])     # flash-attn probed: absent
        sched = SDPA[sched]
    B, fused, chained, row_gemv, kind, lens = PROMPT[sched]
    if _in_child(request, row_gemv):
        return
    dec = _decoder(model, B, bits, fused, chained, row_gemv)
    try:
        truth = _truth_model(dec, SEED)
        spy = dt.Spy(monkeypatch)
        for i, T in enumerate(lens):
            if kind == "rows":
                assert (B * T > 16) == (sched != "P3c")       # P3c: the <= 16-row branch of the blocks
            _call(dec, truth, sched[:2], kind, _ids(B, T, dec.cfg.vocab_size, 20 + i), spy)
    finally:
        dec.unload()


LONG_CASES = [("small", 4), ("hd128", 8)]


@pytest.mark.parametrize("model,bits", LONG_CASES, ids=[f"{m}-q{b}" for m, b in LONG_CASES])
def test_long_prompt_then_decode_across_a_page(model, bits, monkeypatch, request):
    """prefill_rows of 252 tokens, then the benchmarked decode step across position 256: the second page of the permuted
    table."""
    from exllamav2_b200.model import PAGE_SIZE
    if _in_child(request, True):
        return
    dec = _decoder(model, 1, bits)
    try:
        truth = _truth_model(dec, SEED)
        spy = dt.Spy(monkeypatch)
        V = dec.cfg.vocab_size
        _call(dec, truth, "L", "rows", _ids(1, 252, V, 30), spy)
        for t in range(6):
            _call(dec, truth, "L", "decode", _ids(1, 1, V, 40 + t), spy)
        assert dec.pos > PAGE_SIZE
        bt = dec.cache.block_table[0].tolist()
        assert bt[1] != bt[0] + 1
    finally:
        dec.unload()
