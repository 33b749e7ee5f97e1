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
bound per schedule (DESIGN.md §3.6), scaled up only on inputs whose fp16 floor is atypically large (see FLOOR_TYPICAL);
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
import kv_q68

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED = 3
CACHE_LEN = 512         # 2 pages per sequence

# rel-L2 of the decoder's output vs the fp64 truth, per schedule: about 2x the worst measured on an H100 (DESIGN.md §3.6)
OUT_TOL = {"D1": 5e-3, "D2": 5e-3, "D3": 5e-3, "D4": 3e-3, "D5": 9e-3, "D6": 1e-2,
           "P1": 5e-3, "P2": 7e-3, "P3": 6e-3, "P4": 4e-3, "L": 6e-3}
# appended cache rows: |unpack(stored) - truth| <= KV_RATIO * |unpack(pack(fp16(truth))) - truth| + KV_SLACK * |truth|
KV_RATIO = 1.1
KV_SLACK = 2e-3
# The fp16 floor of a call: how far the ideal fp16-storage forward (decoder_truth fp16=True) lies from the exact one on the same
# input.  It is <= FLOOR_TYPICAL on almost every input; where the residual stream cancels it is several times larger, and so is
# any fp16 implementation's error there (on the hd-128 model some decode steps have a floor of 1-2e-2).  The output bound of a
# call scales by floor / FLOOR_TYPICAL above that, and an appended cache row may be off by FLOOR_RATIO x its own floor.
FLOOR_TYPICAL = 3e-3
FLOOR_RATIO = 3.0


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
    for tab, want in ((dec.sin, np.sin(ang)), (dec.cos, np.cos(ang))):
        assert np.abs(tab.float().cpu().numpy() - want).max() <= 1e-3, "RoPE table differs from sin / cos of position x frequency"

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


# ---- cache access -------------------------------------------------------------------------------------------------------

def _snapshot(dec):
    c = dec.cache
    return dict(k=[t.cpu().numpy().copy() for t in c.key_states], ks=[t.cpu().numpy().copy() for t in c.key_scales],
                v=[t.cpu().numpy().copy() for t in c.value_states], vs=[t.cpu().numpy().copy() for t in c.value_scales],
                seqlens=c.cache_seqlens.cpu().numpy().copy(), bt=c.block_table.cpu().numpy().copy())


def _slots(snap, b, lo, hi):
    from exllamav2_b200.model import PAGE_SIZE
    p = np.arange(lo, hi)
    return snap["bt"][b][p // PAGE_SIZE], p % PAGE_SIZE


def _cache_kv(snap, cfg, bits, li, b, lo, hi):
    """Dequantised K and V of sequence b, positions [lo, hi), layer li: [n, KVH, hd] fp64, following the stored page table."""
    n, shp = hi - lo, (hi - lo, cfg.num_kv_heads, cfg.head_dim)
    if n == 0:
        return np.zeros(shp), np.zeros(shp)
    pg, r = _slots(snap, b, lo, hi)
    kb, vb = kv_q68.widths(bits)
    k = kv_q68.kv_unpack(snap["k"][li][pg, r].reshape(n, -1), snap["ks"][li][pg, r].reshape(n, -1), kb)
    v = kv_q68.kv_unpack(snap["v"][li][pg, r].reshape(n, -1), snap["vs"][li][pg, r].reshape(n, -1), vb)
    return k.astype(np.float64).reshape(shp), v.astype(np.float64).reshape(shp)


def _row_err(stored, truth, b):
    """(|stored - truth|, |unpack(pack(fp16(truth))) - truth|, |truth|) per row; rows [n, KVH, hd]."""
    t = truth.reshape(truth.shape[0], -1)
    rq = kv_q68.kv_unpack(*kv_q68.kv_pack(t.astype(np.float16), b), b).astype(np.float64)
    s = stored.reshape(t.shape)
    return np.linalg.norm(s - t, axis=1), np.linalg.norm(rq - t, axis=1), np.linalg.norm(t, axis=1)


# ---- which host branch ran ------------------------------------------------------------------------------------------------

SPIED = ["q_attn_forward_1", "q_attn_forward_1_ex", "paged_attn_decode_q4", "q_mlp_forward_", "q_mlp_forward_ex",
         "q_mlp_forward_rows", "gemv_norm", "gemm_half_q_half_prepared", "gemm_half_q_half", "rms_norm", "q_to_fp16_kv",
         "fp16_to_q_kv"]


class Spy:
    """Records the extension entry points the decoder calls (name, args, kwargs) without changing what they do."""

    def __init__(self, monkeypatch):
        from exllamav2_b200 import ext, model
        self.calls = []
        for name in SPIED:
            monkeypatch.setattr(ext, name, self._wrap(name, getattr(ext, name)))
        monkeypatch.setattr(model, "_sdpa_prefill", self._wrap("_sdpa_prefill", model._sdpa_prefill))
        monkeypatch.setattr(model._lib, "exl2b_paged_attn_decode", self._wrap("exl2b_paged_attn_decode", model._lib.exl2b_paged_attn_decode))

    def _wrap(self, name, fn):
        def w(*a, **kw):
            self.calls.append((name, a, kw))
            return fn(*a, **kw)
        return w

    def take(self):
        c, self.calls = self.calls, []
        return c


def _named(calls, name):
    return [(a, kw) for n, a, kw in calls if n == name]


def _names(calls):
    return {n for n, _, _ in calls}


def _check_branch(sched, kind, calls, dec, L):
    """Assert the host branch a call took, from the entry points it reached."""
    from exllamav2_b200 import ext, model
    B = dec.batch_size
    # above one row the chained schedule runs every matrix on the wgmma kernel: a model with a matrix it cannot stage takes the
    # fused, un-chained branch there instead (D5 as D3 / D6, P1 through q_attn_forward_1)
    staged = all(ext.qmatrix_tc_supported(l.q_handle) for l in dec.linears)
    if not staged and sched == "D5":
        sched = "D6"
    names = _names(calls)
    attn1 = _named(calls, "q_attn_forward_1")
    attn1_ex = _named(calls, "q_attn_forward_1_ex")
    fused = _named(calls, "paged_attn_decode_q4")
    ref_attn = _named(calls, "exl2b_paged_attn_decode")
    rows1 = sorted({a[2] * a[3] for a, _ in attn1})          # batch_size * q_len of q_attn_forward_1
    if sched == "L" and kind == "decode":                    # the long case decodes in the benchmarked step
        sched = "D1"
    if kind == "decode":
        head = {"gemv_norm", "gemm_half_q_half_prepared", "gemm_half_q_half"} & names
        if sched == "D1":
            assert dec.row_gemv and dec.chained and dec.fused_attn and B == 1
            assert len(attn1_ex) == L and all(a[9] is None for a, _ in attn1_ex), "RoPE must be left to the attention kernel"
            assert len(fused) == L and all(kw.get("rope") is not None for _, kw in fused)
            assert head == {"gemv_norm"} and _named(calls, "gemv_norm")[0][1].get("prepared") is True
        elif sched in ("D2", "D5"):
            assert dec.chained and dec.fused_attn and B <= 8 and (B > 1 or not dec.row_gemv)
            assert len(attn1_ex) == L and all(a[9] is not None and a[2] == B for a, _ in attn1_ex)
            assert len(fused) == L and all(kw.get("rope") is None for _, kw in fused)
            assert head == {"gemm_half_q_half_prepared"}
        elif sched in ("D3", "D6"):
            assert dec.fused_attn and not (dec.chained and B <= 8 and staged)
            assert not attn1_ex and rows1 == [B] and len(fused) == L and len(_named(calls, "q_mlp_forward_")) == L
            assert head == {"gemm_half_q_half"} and "rms_norm" in names
            if sched == "D6" and staged:
                assert 8 < B <= 16          # the 9..16-row wgmma, not the many-row path
        elif sched == "D4":
            assert not dec.fused_attn and not fused and len(ref_attn) == L
            assert len(_named(calls, "q_to_fp16_kv")) == L and len(_named(calls, "fp16_to_q_kv")) == L
            assert head == {"gemm_half_q_half"} and "rms_norm" in names
        else:
            raise KeyError(sched)
        return
    if kind == "prefill":
        qlens = [a[3] for a, _ in attn1_ex] + [a[3] for a, _ in attn1]
        if sched == "P1":
            assert dec.chained and dec.fused_attn and B == 1
            if staged:
                assert not attn1 and [a[3] for a, _ in attn1_ex] == [8] * L + [3] * L
            else:
                assert not attn1_ex and [a[3] for a, _ in attn1] == [8] * L + [3] * L
                assert [a[0].shape[1] for a, _ in fused] == [8] * L + [3] * L
            assert "gemv_norm" not in names and "gemm_half_q_half_prepared" not in names
        elif sched == "P2":
            assert dec.fused_attn and B == 3
            assert not attn1_ex and [a[2] * a[3] for a, _ in attn1] == [24] * L + [9] * L   # 24 > 16: gemm_big; 9: wgmma
            assert [a[0].shape[1] for a, _ in fused] == [8] * L + [3] * L
        elif sched == "P4":
            assert not dec.fused_attn and not fused and ref_attn and max(qlens) <= 8
            assert len(_named(calls, "q_to_fp16_kv")) == len(ref_attn) == len(_named(calls, "fp16_to_q_kv"))
        # (prompts of decode schedules run in the decode schedule's flags; their numbers are checked all the same)
        return
    assert kind == "rows"
    assert len(_named(calls, "q_to_fp16_kv")) == L and len(_named(calls, "fp16_to_q_kv")) == L
    assert len(attn1) == L and len(_named(calls, "q_mlp_forward_rows")) == L
    assert len(_named(calls, "_sdpa_prefill")) == (L if model._flash_attn_with_kvcache() is None else 0)


# ---- one call, checked ----------------------------------------------------------------------------------------------------

def _call(dec, truth, sched, kind, ids, spy, chunk=8):
    """Run one decoder call over ids [B, T] and check it against the truth.  Returns the worst output rel-L2."""
    cfg, bits = dec.cfg, dec.cache.wbits
    B, T = ids.shape
    L = cfg.num_layers
    pre = _snapshot(dec)
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
        _check_branch(sched, kind, calls, dec, L)
    post = _snapshot(dec)
    # (3) bookkeeping
    assert np.array_equal(post["seqlens"], pre["seqlens"] + T), (pre["seqlens"], post["seqlens"], T)
    assert dec.pos == pos0 + T
    assert np.array_equal(post["bt"], pre["bt"])
    assert np.isfinite(out).all()
    kb, vb = kv_q68.widths(bits)
    worst, worst_floor, floored = 0.0, 0.0, 0
    chunks = [(t0, min(chunk, T - t0)) for t0 in range(0, T, chunk)] if kind == "prefill" else [(0, T)]
    for b in range(B):
        # (2a) positions written before this call keep their bytes
        pg, r = _slots(pre, b, 0, pos0)
        for key in ("k", "ks", "v", "vs"):
            for li in range(L):
                assert np.array_equal(post[key][li][pg, r], pre[key][li][pg, r]), f"seq {b} layer {li}: {key} of the past changed"
        for t0, n in chunks:
            start = pos0 + t0
            past = [_cache_kv(post, cfg, bits, li, b, 0, start) for li in range(L)]
            pk, pv = [p[0] for p in past], [p[1] for p in past]
            res = truth.forward(ids[b, t0:t0 + n], start, pk, pv)
            res16 = truth.forward(ids[b, t0:t0 + n], start, pk, pv, fp16=True)
            # (2b) the rows this chunk appended
            for li in range(L):
                k, v = _cache_kv(post, cfg, bits, li, b, start, start + n)
                for got, want, want16, wb, what in ((k, res.k[li], res16.k[li], kb, "K"), (v, res.v[li], res16.v[li], vb, "V")):
                    e, eq, nt = _row_err(got, want, wb)
                    floor = np.linalg.norm((want16 - want).reshape(n, -1), axis=1)
                    bad = e > KV_RATIO * eq + np.maximum(KV_SLACK * nt, FLOOR_RATIO * floor)
                    assert not bad.any(), (f"seq {b} layer {li} {what} rows {start + np.flatnonzero(bad)}: error "
                                           f"{e[bad] / nt[bad]} vs quantisation {eq[bad] / nt[bad]}, fp16 floor {floor[bad] / nt[bad]}")
        # (1) output of the call (prefill returns the last chunk's hidden state) against the exact forward, the bound scaled up
        #     where this input's fp16 floor is atypically large
        want, want16 = (res.logits[-1], res16.logits[-1]) if kind == "decode" else (res.hidden, res16.hidden)
        err, floor = oracle.rel_l2(out[b], want), oracle.rel_l2(want16, want)
        bound = OUT_TOL[sched] * max(1.0, floor / FLOOR_TYPICAL)
        floored += bound > OUT_TOL[sched]
        worst, worst_floor = max(worst, err), max(worst_floor, floor)
        assert err <= bound, f"{sched} seq {b}: rel-L2 {err:.3e} vs the fp64 truth (bound {bound:.3e}, fp16 floor {floor:.3e})"
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
        spy = Spy(monkeypatch)
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
    """(4) one step eagerly, then the same step (same cache state) by graph replay: identical logits and cache bytes.  Leaves
    the decoder as it was, with the graph armed, for the checked call that follows."""
    c = dec.cache
    state = [t.clone() for t in (*c.key_states, *c.key_scales, *c.value_states, *c.value_scales, c.cache_seqlens)]

    def restore():
        for dst, src in zip((*c.key_states, *c.key_scales, *c.value_states, *c.value_scales, c.cache_seqlens), state):
            dst.copy_(src)

    g, dec.graph = dec.graph, None
    x = torch.from_numpy(ids).to(DEV)
    spy.take()
    eager = dec.decode(x).clone()
    eager_cache = _snapshot(dec)
    _check_branch("D1", "decode", spy.take(), dec, dec.cfg.num_layers)
    restore()
    dec.pos -= 1
    dec.graph = g
    replay = dec.decode(x).clone()
    replay_cache = _snapshot(dec)
    assert torch.equal(eager.view(torch.int16), replay.view(torch.int16)), "graph replay differs from the eager step"
    for key in ("k", "ks", "v", "vs"):
        for a, b in zip(eager_cache[key], replay_cache[key]):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), f"graph replay stored different {key}"
    assert np.array_equal(eager_cache["seqlens"], replay_cache["seqlens"])
    restore()
    dec.pos -= 1


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
        spy = Spy(monkeypatch)
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
        spy = Spy(monkeypatch)
        V = dec.cfg.vocab_size
        _call(dec, truth, "L", "rows", _ids(1, 252, V, 30), spy)
        for t in range(6):
            _call(dec, truth, "L", "decode", _ids(1, 1, V, 40 + t), spy)
        assert dec.pos > PAGE_SIZE
        bt = dec.cache.block_table[0].tolist()
        assert bt[1] != bt[0] + 1
    finally:
        dec.unload()
