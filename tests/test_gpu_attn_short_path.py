"""Single-token decode attention whose cached rows are all in the staged window (csrc/attn_q4.cu AttnCta::staged_pass):
each warp attends a contiguous range of the CTA's positions with its own running max and sum, and the 8 warps merge once.

The path is taken per CTA when q_len == 1, no ring sub-chunk is streamed and every cached row of the CTA is staged
(c_hi - p_lo <= n_st in tests/attn_regimes.py's plan).  Covered for Q4 / Q6 / Q8 at head dims 64 and 128, MHA and GQA
(32 / 8, 28 / 4), B = 1 and B = 3 with ragged lengths:
  seqlen 0, 1, 127, 128 and stage - 1; split-KV chunks that are all staged; one cached row past the window (the old path).
Inputs: random, zero query (every position weighs the same) and needles at the first and last position of every warp's
range with the appended row as a sink 6 nats above them.  Checked against fp64 attention with the tolerances of
tests/test_gpu_attn_regimes.py (DESIGN.md §3.4), the appended cache bytes against fp16_to_q_kv, a second launch and a
graph replay against the first launch's bits, fused RoPE against RoPE applied first, the chained o_proj row, and (debug
counter 10 of exl2b_debug_set) that exactly the CTAs the plan says take the path took it."""
import ctypes

import numpy as np
import pytest
import torch

import attn_regimes as ar
import test_gpu_attn_regimes as rg

pytestmark = pytest.mark.gpu
DEV = rg.DEV
FMTS = rg.FMTS
HEADS = [(8, 8), (32, 8), (28, 4)]
S0, BETA = rg.S0, rg.BETA


def staged(c):
    """The CTAs of a planned launch that take the warp-local pass (attn_q4.cu AttnCta::all_staged)."""
    return [x for x in c["ctas"] if x["ntail"] == 0 and x["c_hi"] - x["p_lo"] <= x["n_st"]]


def warp_edges(x):
    """First and last position of every warp's range of CTA x (attn_q4.cu AttnCta::staged_pass), cached rows only."""
    tpr = x["hd"] // 32
    g = 32 // tpr
    per = -(-(x["p_hi"] - x["p_lo"]) // (ar.AQ_WARPS * g)) * g
    out = set()
    for w in range(ar.AQ_WARPS):
        lo, hi = x["p_lo"] + w * per, min(x["p_hi"], x["p_lo"] + (w + 1) * per)
        if lo < hi:
            out.update({lo, hi - 1})
    return sorted(p for p in out if p < x["seqlen"])


def split_len(wbits, hd, H):
    """A seqlen for a 2048-position cache at B = 1 whose split-KV chunks are all staged, merged if any such length exists."""
    best = None
    for sl in range(2000, 0, -1):
        p = ar.plan(wbits, hd, H, 1, 1, 2048, [sl])
        if p["nsplit"] > 1 and len(staged(p)) == len(p["ctas"]):
            if len(p["ctas"]) > 1:
                return sl
            best = best or sl
    return best


def case_lens(name, wbits, hd, H):
    """(max_ctx, seqlens) of a case."""
    st = ar.smem_bytes(wbits, hd, 1, 1024, 1)["stage"]
    return {"b1_0": (1024, [0]), "b1_1": (1024, [1]), "b1_127": (1024, [127]), "b1_128": (1024, [128]),
            "b1_stage": (1024, [st - 1]), "b3_ragged": (1024, [st - 1, 0, 127]), "b3_ragged2": (1024, [1, 128, 300 % st]),
            "split": (2048, [split_len(wbits, hd, H)]), "past": (1024, [st + 1])}[name]


NAMES = ["b1_0", "b1_1", "b1_127", "b1_128", "b1_stage", "b3_ragged", "b3_ragged2", "split", "past"]


def build(wbits, hd, H, KVH, name):
    max_ctx, seqlens = case_lens(name, wbits, hd, H)
    B, pps, group = len(seqlens), max_ctx // ar.PAGE, H // KVH
    kb, vb = ar.widths(wbits)
    p = ar.plan(wbits, hd, H, B, 1, max_ctx, seqlens)
    for x in p["ctas"]:
        x["hd"] = hd
    n_staged = len(staged(p))
    if name == "past":
        assert n_staged == 0, p["ctas"]
    else:
        assert n_staged == len(p["ctas"]), p["ctas"]
    if name == "split":
        assert p["nsplit"] > 1, p
    sigma = 1.0 / np.sqrt(hd)
    rng = np.random.default_rng(rg.stable_seed(wbits, hd, H, KVH, name))
    pages_total = B * pps + 1
    bt = rng.permutation(pages_total)[:B * pps].reshape(B, pps).astype(np.int32)
    shp = (pages_total, ar.PAGE, KVH)
    kq = rng.integers(0, 256, size=shp + (hd * kb // 8,), dtype=np.uint8)
    vq = rng.integers(0, 256, size=shp + (hd * vb // 8,), dtype=np.uint8)
    ks = (rng.uniform(0.05, 0.15, size=shp + (hd // 32,)) / (16 if kb == 8 else 1)).astype(np.float16)
    vs = (rng.uniform(0.02, 0.3, size=shp + (hd // 32,)) / (16 if vb == 8 else 1)).astype(np.float16)
    # needles: the first and last cached position of every warp's range, dealt round robin over the heads
    needles = []
    for b in range(B):
        per_head = {}
        edges = sorted({q for x in p["ctas"] if x["b"] == b for q in warp_edges(x)})
        for k, pos in enumerate(edges):
            h = (k + b) % H
            j = per_head.setdefault(h, 0)
            per_head[h] = j + 1
            pg, rr, g = bt[b, pos // ar.PAGE], pos % ar.PAGE, h // group
            kq[pg, rr, g] = ar.s_one_hot_row(hd, kb, rg.ek_of(h, group, hd))
            ks[pg, rr, g, rg.ek_of(h, group, hd) // 32] = rg.key_scale(S0 + 0.25 * (j % 8), sigma, BETA, kb)
            cv = rg.cv_of(j % 8, h, hd)
            vq[pg, rr, g] = ar.s_one_hot_row(hd, vb, cv)
            vs[pg, rr, g, cv // 32] = ar.round8(rng.uniform(0.5, 1.0) * 8 / ar.one_hot_amp(vb))
            needles.append((b, pos, h, j))
    c = dict(plan=p, H=H, KVH=KVH, q_len=1, max_ctx=max_ctx, seqlens=seqlens, B=B, group=group, sigma=sigma, beta=BETA,
             bt=bt, kq=kq, ks=ks, vq=vq, vs=vs, needles=needles, kb=kb, vb=vb, n_staged=n_staged)
    K, V = rg._rows(c, kq, ks, vq, vs)
    return c, K, V


def debug_counter(fn):
    """Run fn() with the attention launch's debug stamps on; debug word 10: CTAs that took the warp-local pass."""
    from exllamav2_b200 import ext as ext_c
    stamps = torch.zeros((64, 32), dtype=torch.int64, device=DEV)
    ext_c.lib.exl2b_debug_set.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
    ext_c.lib.exl2b_debug_set(0, stamps.data_ptr(), 0)
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        ext_c.lib.exl2b_debug_set(0, None, 0)
    return int(stamps[0, 10].item())


@pytest.mark.parametrize("wbits,hd", FMTS)
@pytest.mark.parametrize("H,KVH", HEADS)
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("mode", ["random", "needle", "zero"])
def test_short_path(wbits, hd, H, KVH, name, mode):
    c, K, V = build(wbits, hd, H, KVH, name)
    rng = np.random.default_rng(rg.stable_seed(wbits, hd, H, KVH, name, mode))
    q, kn, vn = rg.make_inputs(c, mode, rng, hd, sink_new=(S0 + 6.0) if mode == "needle" else None)
    out, truth, probs = rg.run_case(c, wbits, hd, q, kn, vn, c["kq"], c["ks"], c["vq"], c["vs"], K, V, ("short", name, wbits, hd, mode))
    if mode == "needle":
        for b in range(c["B"]):
            for h in range(H):
                assert probs[b][0, h][rg.needle_mask(c, b, h)].sum() > 1 - 1e-9, (b, h)
    if mode == "zero":
        for b, sl in enumerate(c["seqlens"]):
            Vb = np.concatenate([V[b], vn[b, :1].astype(np.float64)], 0)
            assert np.allclose(truth[b, 0], np.repeat(Vb.mean(0), c["group"], 0), rtol=1e-9, atol=1e-12)
    if mode == "random":          # the path taken: as many CTAs as the plan names
        n = debug_counter(lambda: rg.launch(c, q, kn, vn, c["kq"], c["ks"], c["vq"], c["vs"]))
        assert n == c["n_staged"] * H, (n, c["n_staged"], H)


def _tensors(c):
    return [rg.t(c[k]) for k in ("kq", "ks", "vq", "vs")]


@pytest.mark.parametrize("wbits,hd", FMTS)
@pytest.mark.parametrize("name", ["b3_ragged", "split"])
def test_short_path_graph_replay(wbits, hd, name):
    """A captured launch replays to the eager launch's output and cache bits."""
    from exllamav2_b200 import ext as ext_c
    c, K, V = build(wbits, hd, 32, 8, name)
    rng = np.random.default_rng(3)
    q, kn, vn = (rg.t(a) for a in rg.make_inputs(c, "random", rng, hd))
    sl, bt = rg.t(np.array(c["seqlens"], dtype=np.int32)), rg.t(c["bt"])
    res = []
    for graph in (False, True):
        kq, ks, vq, vs = _tensors(c)
        out = torch.zeros(q.shape, dtype=torch.half, device=DEV)
        run = lambda: ext_c.paged_attn_decode_q4(q, kn, vn, kq, ks, vq, vs, sl, bt, out, c["sigma"], wbits=wbits)
        if graph:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                run()                                  # warm-up outside the capture (split-KV scratch of stream s)
            torch.cuda.synchronize()
            kq.copy_(rg.t(c["kq"])); ks.copy_(rg.t(c["ks"])); vq.copy_(rg.t(c["vq"])); vs.copy_(rg.t(c["vs"]))
            out.zero_()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                run()
            torch.cuda.synchronize()
            kq.copy_(rg.t(c["kq"])); ks.copy_(rg.t(c["ks"])); vq.copy_(rg.t(c["vq"])); vs.copy_(rg.t(c["vs"]))
            out.zero_()
            g.replay()
        else:
            run()
        torch.cuda.synchronize()
        assert ext_c.paged_attn_status(DEV) == 0
        res.append([x.clone() for x in (out, kq, ks, vq, vs)])
    for a, b in zip(*res):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


@pytest.mark.parametrize("wbits,hd", FMTS)
@pytest.mark.parametrize("H,KVH", [(32, 32), (32, 8), (28, 4)])
@pytest.mark.parametrize("neox", [True, False])
def test_short_path_fused_rope(wbits, hd, H, KVH, neox):
    """Fused RoPE (sin / cos read before the dependency wait) gives the bits of RoPE applied first, output and cache."""
    import exl2_oracle as oracle
    from exllamav2_b200 import ext as ext_c
    c, K, V = build(wbits, hd, H, KVH, "b3_ragged")
    rng = np.random.default_rng(5)
    B = c["B"]
    sin_np, cos_np = oracle.rope_tables(hd, c["max_ctx"])
    sin, cos = rg.t(sin_np), rg.t(cos_np)
    q = rg.t(rng.normal(0, 1, size=(B, 1, H, hd)).astype(np.float16))
    kn = rg.t(rng.normal(0, 1, size=(B, 1, KVH, hd)).astype(np.float16))
    vn = rg.t(rng.normal(0, 1, size=(B, 1, KVH, hd)).astype(np.float16))
    sl, bt = rg.t(np.array(c["seqlens"], dtype=np.int32)), rg.t(c["bt"])

    def run(fused):
        kq, ks, vq, vs = _tensors(c)
        out = torch.zeros((B, 1, H, hd), dtype=torch.half, device=DEV)
        if fused:
            ext_c.paged_attn_decode_q4(q, kn, vn, kq, ks, vq, vs, sl, bt, out, c["sigma"], rope=(sin, cos, 2 if neox else 1), wbits=wbits)
        else:
            qr, kr = q.clone().view(B, 1, H * hd), kn.clone().view(B, 1, KVH * hd)
            ext_c.rope_(qr, sin, cos, -1, H, hd, sl, neox)
            ext_c.rope_(kr, sin, cos, -1, KVH, hd, sl, neox)
            ext_c.paged_attn_decode_q4(qr.view(B, 1, H, hd), kr.view(B, 1, KVH, hd), vn, kq, ks, vq, vs, sl, bt, out, c["sigma"],
                                       wbits=wbits)
        torch.cuda.synchronize()
        return out, kq, ks, vq, vs
    a, b = run(True), run(False)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8))


@pytest.mark.parametrize("wbits", [4, 6, 8])
@pytest.mark.parametrize("name", ["b1_127", "b3_ragged", "split"])
def test_short_path_chained_output(wbits, name):
    """With o_proj as out_consumer the plain output keeps its bits, and o_proj reading the chained row (B = 1: the plain row
    in the matrix's stored order) gives the bits of o_proj over the plain output."""
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200 import synthetic
    from exllamav2_b200.linear import ExLlamaV2Linear
    H, KVH, hd = 32, 8, 128
    c, K, V = build(wbits, hd, H, KVH, name)
    B = c["B"]
    lin = ExLlamaV2Linear(H * hd, 512, device=DEV)
    lin.load(synthetic.random_linear(H * hd, 512, ((4,), (1.0,), 128), device=DEV, seed=4))
    rng = np.random.default_rng(9)
    q, kn, vn = (rg.t(a) for a in rg.make_inputs(c, "random", rng, hd))
    sl, bt = rg.t(np.array(c["seqlens"], dtype=np.int32)), rg.t(c["bt"])
    outs = []
    for oc in (0, lin.q_handle):
        kq, ks, vq, vs = _tensors(c)
        out = torch.zeros((B, 1, H, hd), dtype=torch.half, device=DEV)
        ext_c.paged_attn_decode_q4(q, kn, vn, kq, ks, vq, vs, sl, bt, out, c["sigma"], oc, wbits=wbits)
        torch.cuda.synchronize()
        outs.append((out, kq, ks, vq, vs))
        if oc and B == 1:
            ones = torch.ones(H * hd, dtype=torch.half, device=DEV)
            y_chain = torch.zeros((1, 512), dtype=torch.half, device=DEV)
            y_plain = torch.zeros((1, 512), dtype=torch.half, device=DEV)
            ext_c.gemv_norm(out.view(1, H * hd), lin.q_handle, ones, 1e-6, y_chain, prepared=True)
            ext_c.gemv_norm(out.view(1, H * hd), lin.q_handle, ones, 1e-6, y_plain)
            torch.cuda.synchronize()
            assert torch.equal(y_chain.view(torch.int16), y_plain.view(torch.int16))
    for x, y in zip(*outs):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8))
    lin.unload()
