"""ExLlamaV2Decoder decoding over caches above the single-pass bound of the fused decode attention, so every layer's attention
runs csrc/attn_q4.cu attn_q4_passes_kernel, against the fp64 forward of tests/decoder_truth.py, teacher-forced on the cache.

  hd128   64 heads over 8, hd 128, B = 1, 131 072 positions: the chained single-row schedule (D1: integer GEMV, RoPE inside
          attention, the output chained into o_proj), split-KV chunks of several passes each
  hd64    32 heads over 8, hd 64, B = 9, one page above the single-pass bound (attn_long_plan.largest_fit): the D6 step (two
          wgmma passes, the stand-alone rope_kernel, q_mlp_forward_, rms_norm + gemm head), no split; ragged lengths, from
          single-pass sequences of 1, 256 and 303 positions to ones of two and three passes

The model has 2 layers and a hidden state as wide as its attention (8192).  The cache is filled as bench.py --context fills it (no prompt pass): every (page, row, kv head) of
every layer is a copy of one row of a pool of random rows, and cache_seqlens is set directly.  The truth reads the pool's
rows dequantised exactly (kv_q68.kv_unpack_exact), as the fused attention reads them.  The starting lengths are taken
from tests/attn_long_plan.py so that the steps cross the point where each split-KV chunk gains a pass; each step reads the rows the steps before it appended.

Each decode step runs eagerly, then the decoder is captured and further steps run by graph replay, each first checked to give
the eager step's bits (decoder_truth.graph_matches_eager).  Per step: the branch (decoder_truth.check_branch on the entry
points reached, and every attention launch in the passes regime); seqlens advanced by one; every cache byte except the
appended rows unchanged; each appended row within decoder_truth's K/V bound of the fp64 row; the logits of every sequence
within OUT_TOL[schedule] of the fp64 truth, scaled by the fp16 floor as decoder_truth.check_call scales it.  The truth reads
the past rows (the pool's rows, and the rows the decoder appended) exactly dequantised."""
import numpy as np
import pytest
import torch

import attn_long_plan as alp
import attn_regimes as ar
import decoder_truth as dt
import kv_q68
from exl2_oracle import rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED = 7
POOL = 2048
MEASURED = {}


B_OF = {"hd128": 1, "hd64": 9}
SCHED_OF = {"hd128": "D1", "hd64": "D6"}


def _cfg(model, bits):
    from exllamav2_b200.model import PRESETS, LlamaConfig
    plan = PRESETS["test-small"]().plan
    # the attention is as wide as the hidden state, as in Llama-2-70B, whose heads the hd128 model has
    if model == "hd128":
        return LlamaConfig("long-h64-kv8-hd128", 8192, 4096, 64, 8, 128, 2, 1024, max_seq_len=131072, plan=plan)
    assert model == "hd64"
    cap = alp.largest_fit(bits, 64, 32, B_OF[model]) + ar.PAGE
    return LlamaConfig("long-h32-kv8-hd64", 2048, 4096, 32, 8, 64, 2, 1024, max_seq_len=cap, plan=plan)


def _start_lengths(model, bits, cfg, B, steps):
    """Lengths at which the steps cross the edges the passes regime has (see the module docstring)."""
    cap, hd, H = cfg.max_seq_len, cfg.head_dim, cfg.num_heads
    lp = alp.long_plan(bits, hd, H, B, 1, cap)
    pl = lp["pass_len"]
    if model == "hd64":           # no split: single-pass sequences, and ones that gain their second / third pass mid-way
        return [1, 256, 303, 0, 257, pl - 2, pl + 1, 2 * pl - 1, cap - steps]
    k = (cap // lp["nsplit"]) // pl                      # a chunk of k * pl positions gains its (k + 1)-th pass one step later
    return [lp["nsplit"] * k * pl - 3]


class Pool:
    """Per layer: the stored rows the cache is made of (random rows, then each row a step appended), their oracle
    dequantisation, and which of them every (page, row, kv head) holds."""

    def __init__(self, dec, rng):
        c, self.bits = dec.cache, dec.cache.wbits
        self.kb, self.vb = kv_q68.widths(self.bits)
        hd, KVH = dec.cfg.head_dim, dec.cfg.num_kv_heads
        self.layers = []
        for li in range(dec.cfg.num_layers):
            kq = rng.integers(0, 256, size=(POOL, hd * self.kb // 8), dtype=np.uint8)
            vq = rng.integers(0, 256, size=(POOL, hd * self.vb // 8), dtype=np.uint8)
            # element scales of a row of std ~0.3 (keys) / ~0.5 (values) once dequantised, as bench.py --context's fixed 0.35
            ks = (rng.uniform(0.2, 0.5, size=(POOL, hd // 32)) / (16 if self.kb == 8 else 1)).astype(np.float16)
            vs = (rng.uniform(0.3, 0.8, size=(POOL, hd // 32)) / (16 if self.vb == 8 else 1)).astype(np.float16)
            idx = rng.integers(0, POOL, size=tuple(c.key_states[li].shape[:3]), dtype=np.int64)
            L = dict(rows=[kq, ks, vq, vs], idx=idx)
            L["kd"] = kv_q68.kv_unpack_exact(kq, ks, self.kb)
            L["vd"] = kv_q68.kv_unpack_exact(vq, vs, self.vb)
            self.layers.append(L)
            for dst, src in zip((c.key_states[li], c.key_scales[li], c.value_states[li], c.value_scales[li]), self.expected(li)):
                dst.copy_(src)

    def expected(self, li):
        """The layer's cache tensors as the pool says they are."""
        L = self.layers[li]
        idx = torch.from_numpy(L["idx"]).to(DEV)
        return [torch.from_numpy(a).to(DEV)[idx] for a in L["rows"]]

    def past(self, li, bt, b, n):
        """Dequantised K and V of sequence b, positions [0, n): [n, KVH, hd] fp64."""
        from exllamav2_b200.model import PAGE_SIZE
        L = self.layers[li]
        p = np.arange(n)
        sel = L["idx"][bt[b, p // PAGE_SIZE], p % PAGE_SIZE]
        return L["kd"][sel], L["vd"][sel]

    def adopt(self, li, cache, slots):
        """Rows a step appended at slots [(page, row)] (every kv head) become pool rows; returns their dequantised K, V."""
        L = self.layers[li]
        got = []
        for t in (cache.key_states[li], cache.key_scales[li], cache.value_states[li], cache.value_scales[li]):
            got.append(np.stack([t[pg, r].cpu().numpy() for pg, r in slots]))      # [n, KVH, ...]
        n, KVH = got[0].shape[:2]
        base = L["rows"][0].shape[0]
        for j in range(4):
            L["rows"][j] = np.concatenate([L["rows"][j], got[j].reshape(n * KVH, -1)])
        kd = kv_q68.kv_unpack_exact(got[0].reshape(n * KVH, -1), got[1].reshape(n * KVH, -1), self.kb)
        vd = kv_q68.kv_unpack_exact(got[2].reshape(n * KVH, -1), got[3].reshape(n * KVH, -1), self.vb)
        L["kd"], L["vd"] = np.concatenate([L["kd"], kd]), np.concatenate([L["vd"], vd])
        for i, (pg, r) in enumerate(slots):
            L["idx"][pg, r] = base + i * KVH + np.arange(KVH)
        return kd.reshape(n, KVH, -1), vd.reshape(n, KVH, -1)


def _truth(dec):
    cfg = dec.cfg
    W = [l.get_weight_tensor_dq() for l in dec.linears]
    layers = [dt.TruthLayer(L.input_norm, L.post_norm, *W[7 * li:7 * li + 7]) for li, L in enumerate(dec.layers)]
    return dt.TorchTruthModel(layers, dec.final_norm, W[-1], dec.embed, dec.sin, dec.cos, cfg.num_heads, cfg.num_kv_heads,
                              cfg.head_dim, cfg.norm_eps, DEV)


def _check_passes(calls, dec):
    """Every attention launch of the step ran in the passes regime (tests/attn_long_plan.py)."""
    launches = dt.named(calls, "paged_attn_decode_q4")
    assert len(launches) == dec.cfg.num_layers
    for a, kw in launches:
        B, q_len, H, hd = a[0].shape
        page, pps = a[3].shape[1], a[8].shape[1]
        assert alp.long_plan(dec.cache.wbits, hd, H, B, q_len, page * pps)["passes"]


def _eager_branch(calls, dec, sched):
    dt.check_branch(sched, "decode", calls, dec, dec.cfg.num_layers)
    _check_passes(calls, dec)


# hd64: the reference op sequence (q_to_fp16_kv -> fp16 attention -> fp16_to_q_kv) on the same state bounds the step as well.
# On these inputs the logits are ill-conditioned far beyond what the fp16 floor measures (DESIGN.md §3.9): over 177 sequence
# outputs of a grid of batch sizes, lengths, capacities and pasts, the reference sequence reached 1.6e-2 at floors of 1e-3,
# and the fused step was at most 1.78x the reference's error.  A fused step may be REF_RATIO x as far from the truth as the
# reference sequence on the same state; a fault in the fused path shows as a fused error far above the reference's.
REF_RATIO = {"hd64": 3.0}


def _reference_logits(dec, ids):
    """The logits of the same decode step through the reference op sequence, on the same cache state; the decoder is left
    as it was (state, position and graph)."""
    c = dec.cache
    live = (*c.key_states, *c.key_scales, *c.value_states, *c.value_scales, c.cache_seqlens)
    state = [t.clone() for t in live]
    g, dec.graph, dec.fused_attn = dec.graph, None, False
    try:
        out = dec.decode(torch.from_numpy(ids).to(DEV)).float().cpu().numpy()
        torch.cuda.synchronize()
    finally:
        for d, src in zip(live, state):
            d.copy_(src)
        dec.graph, dec.fused_attn = g, True
        dec.pos -= 1
    return out


def _step(dec, truth, pool, sched, ids, spy, tag, ref_ratio=0.0):
    """One checked decode step (eager, or by replay when the decoder is captured)."""
    from exllamav2_b200.model import PAGE_SIZE
    cfg, c = dec.cfg, dec.cache
    B, L = dec.batch_size, cfg.num_layers
    sl0 = c.cache_seqlens.cpu().numpy().copy()
    bt = c.block_table.cpu().numpy().copy()
    pos0 = dec.pos
    ref = _reference_logits(dec, ids) if ref_ratio else None
    spy.take()
    out = dec.decode(torch.from_numpy(ids).to(DEV)).float().cpu().numpy()
    torch.cuda.synchronize()
    calls = spy.take()
    if dec.graph is None:                    # (a replayed step reaches no entry point: its eager twin is checked instead)
        dt.check_branch(sched, "decode", calls, dec, L)
        _check_passes(calls, dec)
    assert np.array_equal(c.cache_seqlens.cpu().numpy(), sl0 + 1) and dec.pos == pos0 + 1
    assert np.array_equal(c.block_table.cpu().numpy(), bt)
    slots = [(int(bt[b, s // PAGE_SIZE]), int(s % PAGE_SIZE)) for b, s in enumerate(sl0)]
    # every cache byte but the appended rows is the pool's
    for li in range(L):
        want = pool.expected(li)
        for w, got in zip(want, (c.key_states[li], c.key_scales[li], c.value_states[li], c.value_scales[li])):
            for pg, r in slots:
                w[pg, r] = got[pg, r]
            assert torch.equal(w.view(torch.uint8), got.view(torch.uint8)), f"{tag} layer {li}: a cache byte moved"
    past = [[pool.past(li, bt, b, int(sl0[b])) for li in range(L)] for b in range(B)]
    new = [pool.adopt(li, c, slots) for li in range(L)]
    worst = 0.0
    for b in range(B):
        pk, pv = [p[0] for p in past[b]], [p[1] for p in past[b]]
        res = truth.forward(ids[b], int(sl0[b]), pk, pv)
        res16 = truth.forward(ids[b], int(sl0[b]), pk, pv, fp16=True)
        for li in range(L):
            for got, want, want16, wb, what in ((new[li][0][b:b + 1], res.k[li], res16.k[li], pool.kb, "K"),
                                                (new[li][1][b:b + 1], res.v[li], res16.v[li], pool.vb, "V")):
                e, eq, nt = dt.row_err(got, want, wb)
                floor = np.linalg.norm((want16 - want).reshape(1, -1), axis=1)
                assert not (e > dt.KV_RATIO * eq + np.maximum(dt.KV_SLACK * nt, dt.FLOOR_RATIO * floor)).any(), \
                    (tag, b, li, what, e / nt, eq / nt, floor / nt)
        err, floor = rel_l2(out[b], res.logits[-1]), rel_l2(res16.logits[-1], res.logits[-1])
        bound = dt.OUT_TOL[sched] * max(1.0, floor / dt.FLOOR_TYPICAL)
        err_ref = rel_l2(ref[b], res.logits[-1]) if ref is not None else 0.0
        bound = max(bound, ref_ratio * err_ref)
        print(f"  {tag} seq {b} (seqlen {sl0[b]}): rel-L2 {err:.3e}, reference sequence {err_ref:.3e}, floor {floor:.3e}")
        assert err <= bound, (f"{tag} seq {b} (seqlen {sl0[b]}): rel-L2 {err:.3e} (bound {bound:.3e}, fp16 floor {floor:.3e}, "
                              f"reference sequence {err_ref:.3e})")
        worst = max(worst, err)
    MEASURED[tag] = max(MEASURED.get(tag, 0.0), worst)
    print(f"TRUTH long {tag} seqlens {sl0.min()}..{sl0.max()}: logits rel-L2 {worst:.3e}")


CASES = [("hd128", 4), ("hd128", 8), ("hd64", 4), ("hd64", 6), ("hd64", 8)]


@pytest.mark.parametrize("model,bits", CASES, ids=[f"{m}-q{b}" for m, b in CASES])
def test_decode_long_cache_vs_fp64(model, bits, monkeypatch):
    from exllamav2_b200.model import ExLlamaV2Decoder
    cfg = _cfg(model, bits)
    B, sched = B_OF[model], SCHED_OF[model]
    steps = 2
    dec = ExLlamaV2Decoder(cfg, device=DEV, seed=SEED, batch_size=B, cache_len=cfg.max_seq_len, cache_bits=bits)
    try:
        assert not alp.long_plan(bits, cfg.head_dim, cfg.num_heads, B, 1, alp.largest_fit(bits, cfg.head_dim, cfg.num_heads, B))["passes"]
        assert cfg.max_seq_len > alp.largest_fit(bits, cfg.head_dim, cfg.num_heads, B)
        if sched == "D1":
            assert dec.row_gemv, "the library was loaded with EXL2B_GEMV=tc"
        bt = dec.cache.block_table           # every sequence's pages scattered over the pool
        perm = torch.randperm(bt.numel(), generator=torch.Generator().manual_seed(3000 + bits)).to(torch.int32)
        bt.copy_(perm.view(bt.shape).to(bt.device))
        rng = np.random.default_rng(SEED * 10 + bits)
        pool = Pool(dec, rng)
        lens = _start_lengths(model, bits, cfg, B, 2 * steps)
        dec.cache.cache_seqlens.copy_(torch.tensor(lens, dtype=torch.int32, device=DEV))
        dec.pos = max(lens)
        truth = _truth(dec)
        spy = dt.Spy(monkeypatch)
        V = cfg.vocab_size
        ids = lambda t: rng.integers(0, V, size=(B, 1)).astype(np.int64)
        for t in range(steps):
            _step(dec, truth, pool, sched, ids(t), spy, f"{model} Q{bits} eager", REF_RATIO.get(model, 0.0))
        dec.capture()
        for t in range(steps):
            x = ids(t)
            spy.take()
            dt.graph_matches_eager(dec, x, lambda: _eager_branch(spy.take(), dec, sched))
            _step(dec, truth, pool, sched, x, spy, f"{model} Q{bits} graph", REF_RATIO.get(model, 0.0))
    finally:
        dec.unload()
        torch.cuda.empty_cache()
