"""Single-token decode attention over caches whose score buffer does not fit shared memory in one pass (csrc/attn_q4.cu
attn_q4_passes_kernel), for Q4 / Q6 / Q8 at head dims 64 and 128, against fp64 softmax attention over the
oracle-dequantised cache plus the unquantised new row.

The cases, each a capacity tests/attn_long_plan.py puts in the passes regime (asserted):
  batched   32 heads over 8, B = 9, no split, ragged lengths, capacity one page above the single-pass bound
  gqa7      28 heads over 4, B = 10, no split, capacity one page above the bound
  split     64 heads over 8, B = 1, the full cache: split-KV chunks of several passes each (131072 positions at hd 128,
            262144 at hd 64, where 131072 still fits one pass)
  short     64 heads over 8, B = 1, 300 positions in that cache: one pass, one chunk

Inputs (`mode`): random; zero query (the mean of every value row); needle (both sides of every pass, chunk, ring sub-chunk and
page edge of the plan are needles of one head each, 40 nats above the background, plus the appended row); rise / fall (two more
needles per head in every chunk, in its first and its last pass, the later one 6 nats above the earlier (rise) or below it
(fall), so the running max changes between passes); sink (the appended row 6 nats above every cached needle).

The cache is built on the device from a pool of random rows (each cached row is a copy of one pool row; needles are pool
rows of their own), so the oracle dequantises only the pool, and the truth gathers the pool in fp64 on the device.
Every case checks the output per (b, h) against TOL of test_gpu_attn_regimes.py, that the appended rows are this library's
fp16_to_q_kv bytes and nothing else moved, that a second launch gives the same bits, and that the status word is 0.
"""
import functools
import zlib

import numpy as np
import pytest
import torch

import attn_long_plan as alp
import attn_regimes as ar
import exl2_oracle as oracle
import kv_q68

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FMTS = [(w, hd) for w in (4, 6, 8) for hd in (64, 128)]
TOL = dict(rel=1.6e-3, mx=2.5e-3)          # test_gpu_attn_regimes.py TOL
S0, BETA = 40.0, 16.0                      # needle score above a zero score (nats); needle query amplitude
POOL = 4096
MEASURED = {}


def seed_of(*key):
    return zlib.crc32(repr(key).encode())


def shape(name, wbits, hd):
    """(H, KVH, B, capacity, seqlens) of a case."""
    if name in ("batched", "gqa7"):
        H, KVH, B = (32, 8, 9) if name == "batched" else (28, 4, 10)
        cap = alp.largest_fit(wbits, hd, H, B) + ar.PAGE
        pl = alp.long_plan(wbits, hd, H, B, 1, cap)["pass_len"]
        sl = [cap - 1, 0, 1, pl - 1, pl, pl + 1, 2 * pl + 135, cap // 2 + 77, cap - 300, cap - 2][:B]
        return H, KVH, B, cap, sl
    cap = 131072 if hd == 128 else 262144
    return 64, 8, 1, cap, [cap - 1] if name == "split" else [300]


def ek_of(h, group, hd):
    return ((h % group) * 37 + 3) % hd


def cv_of(j, h, hd):
    return (j * (hd // 8) + 3 * h) % hd


def key_scale(score, sigma, bits):
    return ar.round8(score / (sigma * BETA * ar.one_hot_amp(bits)))


@functools.lru_cache(maxsize=1)
def base_case(wbits, hd, name):
    """Plan, block table, row pool, the pool index of every cached (page, row, kv head), and the needle map."""
    H, KVH, B, cap, seqlens = shape(name, wbits, hd)
    kb, vb = ar.widths(wbits)
    lp = alp.long_plan(wbits, hd, H, B, 1, cap, seqlens)
    assert lp["passes"] and lp["fits"], (name, wbits, hd)
    if name == "split":
        assert lp["nsplit"] > 1 and all(len(c["passes"]) > 1 for c in lp["ctas"])
    if name == "short":
        assert [len(c["passes"]) for c in lp["ctas"]] == [1]
    if name in ("batched", "gqa7"):
        assert lp["nsplit"] == 1 and max(len(c["passes"]) for c in lp["ctas"]) > 1
    rng = np.random.default_rng(seed_of(wbits, hd, name))
    pps, group, sigma = cap // ar.PAGE, H // KVH, 1.0 / np.sqrt(hd)
    pages_total = B * pps + 1                      # one page no sequence owns
    bt = rng.permutation(pages_total)[:B * pps].reshape(B, pps).astype(np.int32)
    kq = [rng.integers(0, 256, size=(POOL, hd * kb // 8), dtype=np.uint8)]
    vq = [rng.integers(0, 256, size=(POOL, hd * vb // 8), dtype=np.uint8)]
    ks = [(rng.uniform(0.05, 0.15, size=(POOL, hd // 32)) / (16 if kb == 8 else 1)).astype(np.float16)]
    vs = [(rng.uniform(0.02, 0.3, size=(POOL, hd // 32)) / (16 if vb == 8 else 1)).astype(np.float16)]
    idx = rng.integers(0, POOL, size=(pages_total, ar.PAGE, KVH), dtype=np.int64)
    c = dict(H=H, KVH=KVH, B=B, cap=cap, seqlens=seqlens, kb=kb, vb=vb, lp=lp, group=group, sigma=sigma, bt=bt, idx=idx,
             pool=[kq, ks, vq, vs], needles=[], taken=set())
    for b in range(B):
        per_head = {}
        for k, pos in enumerate(alp.boundary_positions(lp, b)):
            h = (k + b) % H
            j = per_head.setdefault(h, 0)
            per_head[h] = j + 1
            add_needle(c, b, pos, h, S0 + 0.25 * (j % 8), j, rng)
    return c


def add_needle(c, b, pos, h, score, j, rng):
    """Position pos of sequence b becomes a pool row of its own: head h's one-hot key scoring `score`, a one-hot value."""
    hd = c["pool"][1][0].shape[1] * 32
    kq, ks, vq, vs = c["pool"]
    ek, cv = ek_of(h, c["group"], hd), cv_of(j % 8, h, hd)
    ksr = np.full((1, hd // 32), 0.1 / (16 if c["kb"] == 8 else 1), np.float16)
    ksr[0, ek // 32] = key_scale(score, c["sigma"], c["kb"])
    vsr = np.full((1, hd // 32), 0.1 / (16 if c["vb"] == 8 else 1), np.float16)
    vsr[0, cv // 32] = ar.round8(rng.uniform(0.5, 1.0) * 8 / ar.one_hot_amp(c["vb"]))
    kq.append(ar.s_one_hot_row(hd, c["kb"], ek)[None])
    ks.append(ksr)
    vq.append(ar.s_one_hot_row(hd, c["vb"], cv)[None])
    vs.append(vsr)
    pg, rr = c["bt"][b, pos // ar.PAGE], pos % ar.PAGE
    c["idx"][pg, rr, h // c["group"]] = POOL + len(kq) - 2     # kq: the POOL-row array, then one row per needle
    c["needles"].append((b, pos, h))
    c["taken"].add((b, pos))


def skewed(c0, mode, hd):
    """rise / fall: per chunk and head, a needle in the first pass and one in the last pass, 6 nats apart."""
    c = dict(c0, pool=[list(a) for a in c0["pool"]], idx=c0["idx"].copy(), needles=list(c0["needles"]),
             taken=set(c0["taken"]))
    rng = np.random.default_rng(seed_of(mode))
    for cta in c["lp"]["ctas"]:
        b, sl = cta["b"], cta["seqlen"]
        first, last = cta["passes"][0], cta["passes"][-1]
        for h in range(c["H"]):
            for ps, hi_score, start in ((first, mode == "fall", first["lo"] + 20 + 3 * h),
                                        (last, mode == "rise", min(last["hi"], sl) - 2 - 3 * h)):
                pos = start
                while (b, pos) in c["taken"]:
                    pos += 1
                if ps["lo"] <= pos < min(ps["hi"], sl):
                    add_needle(c, b, pos, h, S0 + (6.0 if hi_score else 0.0), 1, rng)
    return c


def device_cache(c):
    kq, ks, vq, vs = (torch.from_numpy(np.concatenate(a)).to(DEV) for a in c["pool"])
    idx = torch.from_numpy(c["idx"]).to(DEV)
    return kq[idx].contiguous(), ks[idx].contiguous(), vq[idx].contiguous(), vs[idx].contiguous()


def make_inputs(c, mode, rng, hd):
    B, H, KVH, group = c["B"], c["H"], c["KVH"], c["group"]
    kn = rng.normal(0, 1, size=(B, 1, KVH, hd)).astype(np.float16)
    vn = rng.normal(0, 1, size=(B, 1, KVH, hd)).astype(np.float16)
    if mode == "random":
        return rng.normal(0, 4, size=(B, 1, H, hd)).astype(np.float16), kn, vn
    if mode == "zero":
        return np.zeros((B, 1, H, hd), np.float16), kn, vn
    q = np.zeros((B, 1, H, hd), np.float16)
    kn[:] = 0
    for h in range(H):
        d = ar.key_direction(hd, c["kb"], ek_of(h, group, hd))
        q[:, :, h] = (BETA * np.sign(d)).astype(np.float16)
        s = key_scale(S0 + (6.0 if mode == "sink" else 1.0), c["sigma"], c["kb"])
        kn[:, 0, h // group] = (kn[:, 0, h // group].astype(np.float64) + d * float(s)).astype(np.float16)
    return q, kn, vn


def truth(c, q, kn, vn, return_mass=False):
    """fp64 attention on the device: the cached rows are the oracle-dequantised pool rows, gathered."""
    kd = [torch.from_numpy(kv_q68.kv_unpack(np.concatenate(c["pool"][0]), np.concatenate(c["pool"][1]), c["kb"]).astype(np.float64)).to(DEV)]
    vd = [torch.from_numpy(kv_q68.kv_unpack(np.concatenate(c["pool"][2]), np.concatenate(c["pool"][3]), c["vb"]).astype(np.float64)).to(DEV)]
    idx, bt = torch.from_numpy(c["idx"]).to(DEV), torch.from_numpy(c["bt"]).to(DEV).long()
    B, H, KVH, g = c["B"], c["H"], c["KVH"], c["group"]
    hd = q.shape[-1]
    out = np.zeros((B, 1, H, hd))
    mass = []
    for b, sl in enumerate(c["seqlens"]):
        p = torch.arange(sl, device=DEV)
        rows = idx[bt[b, p // ar.PAGE], p % ar.PAGE]                                  # [sl, KVH]
        K = torch.cat([kd[0][rows], torch.from_numpy(kn[b]).to(DEV).double()], 0)    # [sl + 1, KVH, hd]
        V = torch.cat([vd[0][rows], torch.from_numpy(vn[b]).to(DEV).double()], 0)
        qb = torch.from_numpy(q[b, 0]).to(DEV).double().view(KVH, g, hd)
        s = torch.einsum("kgd,nkd->kgn", qb, K) * c["sigma"]
        pr = torch.softmax(s, -1)
        out[b, 0] = torch.einsum("kgn,nkd->kgd", pr, V).reshape(H, hd).cpu().numpy()
        if return_mass:
            m = np.zeros((H, sl + 1), dtype=bool)
            for (bb, pos, h) in c["needles"]:
                if bb == b:
                    m[h, pos] = True
            m[:, sl] = True
            mass.append(float((pr.reshape(H, sl + 1) * torch.from_numpy(m).to(DEV)).sum(-1).min()))
    return (out, mass) if return_mass else out


def launch(c, q, kn, vn, cache, out_consumer=0, rope=None, out=None):
    from exllamav2_b200 import ext as ext_c
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV) if isinstance(a, np.ndarray) else a
    out = torch.zeros(q.shape, dtype=torch.half, device=DEV) if out is None else out
    ext_c.paged_attn_decode_q4(t(q), t(kn), t(vn), *cache, t(np.array(c["seqlens"], dtype=np.int32)), t(c["bt"]), out,
                               c["sigma"], out_consumer, rope=rope, wbits={(4, 4): 4, (8, 4): 6, (8, 8): 8}[(c["kb"], c["vb"])])
    torch.cuda.synchronize()
    assert ext_c.paged_attn_status(DEV) == 0
    return out


def check_cache(c, kn, vn, before, after, wbits):
    """The appended rows are fp16_to_q_kv's bytes; every other byte is as it was."""
    from exllamav2_b200 import ext as ext_c
    B, KVH = c["B"], c["KVH"]
    hd = kn.shape[-1]
    n = B * KVH
    npad = -(-n * hd // 512) * 512 // hd

    def pad(x):
        z = torch.zeros((1, 1, npad, hd), dtype=torch.half, device=DEV)
        z.view(npad, hd)[:n] = torch.from_numpy(x).to(DEV).view(n, hd)
        return z
    pk = torch.zeros((1, 1, npad, hd * c["kb"] // 8), dtype=torch.uint8, device=DEV)
    pv = torch.zeros((1, 1, npad, hd * c["vb"] // 8), dtype=torch.uint8, device=DEV)
    pks, pvs = (torch.zeros((1, 1, npad, hd // 32), dtype=torch.half, device=DEV) for _ in range(2))
    ext_c.fp16_to_q_kv(pad(kn), pk, pks, pad(vn), pv, pvs, 1, 0, 1, 0, ext_c.none_tensor, ext_c.none_tensor, wbits)
    want = [a.clone() for a in before]
    for b, sl in enumerate(c["seqlens"]):
        pg, rr = int(c["bt"][b, sl // ar.PAGE]), sl % ar.PAGE
        for w, src in zip(want, (pk, pks, pv, pvs)):
            w[pg, rr] = src.view(npad, -1)[b * KVH:(b + 1) * KVH]
    for w, a in zip(want, after):
        assert torch.equal(w.view(torch.uint8), a.view(torch.uint8))


def compare(got, want, tag):
    g = got.astype(np.float64)
    assert np.isfinite(g).all(), tag
    rel = np.linalg.norm(g - want, axis=-1) / np.maximum(np.linalg.norm(want, axis=-1), 1e-300)
    mx = np.abs(g - want).max(-1) / np.maximum(np.abs(want).max(-1), 1e-30)
    old = MEASURED.get(tag, (0.0, 0.0))
    MEASURED[tag] = (max(old[0], float(rel.max())), max(old[1], float(mx.max())))
    bad = np.argwhere((rel > TOL["rel"]) | (mx > TOL["mx"]))
    assert len(bad) == 0, (tag, [(tuple(x), rel[tuple(x)], mx[tuple(x)]) for x in bad[:8]])


MODES = ["random", "zero", "needle", "rise", "fall", "sink"]
CASES = [(w, hd, n, m) for (w, hd) in FMTS for n in ("batched", "gqa7", "split", "short") for m in MODES
         if not (n == "short" and m in ("rise", "fall"))]


@pytest.mark.parametrize("wbits,hd,name,mode", CASES)
def test_long_context(wbits, hd, name, mode):
    c = base_case(wbits, hd, name)
    if mode in ("rise", "fall"):
        c = skewed(c, mode, hd)
    rng = np.random.default_rng(seed_of(wbits, hd, name, mode))
    q, kn, vn = make_inputs(c, mode, rng, hd)
    before = device_cache(c)
    cache = [a.clone() for a in before]
    out = launch(c, q, kn, vn, cache).cpu().numpy()
    check_cache(c, kn, vn, before, cache, wbits)
    want, mass = truth(c, q, kn, vn, return_mass=True)
    if mode not in ("random", "zero"):
        assert min(mass) > 1 - 1e-9, mass             # the design: the needles carry all but ~1e-9 of every head's mass
    compare(out, want, (name, wbits, hd, mode))
    out2 = launch(c, q, kn, vn, cache).cpu().numpy()
    assert np.array_equal(out.view(np.uint16), out2.view(np.uint16)), "a second identical launch gave different bits"


# ---- o_proj reading the output, fused RoPE, a captured launch --------------------------------------------------------

def small_case(wbits, hd, H, KVH, B, cap, seqlens, seed):
    kb, vb = ar.widths(wbits)
    rng = np.random.default_rng(seed)
    pages_total = B * (cap // ar.PAGE)
    kq = [rng.integers(0, 256, size=(POOL, hd * kb // 8), dtype=np.uint8)]
    vq = [rng.integers(0, 256, size=(POOL, hd * vb // 8), dtype=np.uint8)]
    ks = [(rng.uniform(0.05, 0.15, size=(POOL, hd // 32)) / (16 if kb == 8 else 1)).astype(np.float16)]
    vs = [(rng.uniform(0.02, 0.3, size=(POOL, hd // 32)) / (16 if vb == 8 else 1)).astype(np.float16)]
    c = dict(H=H, KVH=KVH, B=B, cap=cap, seqlens=seqlens, kb=kb, vb=vb, group=H // KVH, sigma=1.0 / np.sqrt(hd),
             bt=rng.permutation(pages_total).reshape(B, -1).astype(np.int32), pool=[kq, ks, vq, vs], needles=[],
             idx=rng.integers(0, POOL, size=(pages_total, ar.PAGE, KVH), dtype=np.int64))
    q = rng.normal(0, 4, size=(B, 1, H, hd)).astype(np.float16)
    kn = rng.normal(0, 1, size=(B, 1, KVH, hd)).astype(np.float16)
    vn = rng.normal(0, 1, size=(B, 1, KVH, hd)).astype(np.float16)
    return c, q, kn, vn


@pytest.mark.parametrize("wbits", [4, 6, 8])
@pytest.mark.parametrize("H,B", [(64, 1), (32, 8)])
def test_chained_output_read_by_o_proj(wbits, H, B):
    """out_consumer = o_proj in the passes regime: one row (64 heads, 131072 positions, split) left as the single-row GEMV's
    plain row, 8 rows (32 heads, one page above the bound, no split) in the core-matrix layout; o_proj on that buffer equals
    o_proj on the plain output bit for bit, and the output is right."""
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200 import synthetic
    from exllamav2_b200.linear import ExLlamaV2Linear
    hd, KVH = 128, 8
    cap = 131072 if B == 1 else alp.largest_fit(wbits, hd, H, B) + ar.PAGE
    seqlens = [cap - 1 - 977 * b for b in range(B)]
    assert alp.long_plan(wbits, hd, H, B, 1, cap)["passes"]
    c, q, kn, vn = small_case(wbits, hd, H, KVH, B, cap, seqlens, seed=wbits * 10 + B)
    lin = ExLlamaV2Linear(H * hd, 512, device=DEV)
    lin.load(synthetic.random_linear(H * hd, 512, ((4,), (1.0,), 128), device=DEV, seed=4))
    out = launch(c, q, kn, vn, device_cache(c), out_consumer=lin.q_handle)
    y_chain = torch.zeros((B, 512), dtype=torch.half, device=DEV)
    y_plain = torch.zeros((B, 512), dtype=torch.half, device=DEV)
    x = out.view(B, H * hd)
    if B == 1:
        w = torch.ones(H * hd, dtype=torch.half, device=DEV)
        ext_c.gemv_norm(x, lin.q_handle, w, 1e-6, y_chain, prepared=True)
        ext_c.gemv_norm(x, lin.q_handle, w, 1e-6, y_plain)
    else:
        ext_c.gemm_half_q_half_prepared(lin.q_handle, y_chain, False, 0.0)
        ext_c.gemm_half_q_half(x, lin.q_handle, y_plain)
    torch.cuda.synchronize()
    assert torch.equal(y_chain.view(torch.int16), y_plain.view(torch.int16))
    compare(out.cpu().numpy(), truth(c, q, kn, vn), ("chain", wbits, hd, f"B{B}"))
    lin.unload()


@pytest.mark.parametrize("wbits,hd", FMTS)
@pytest.mark.parametrize("neox", [True, False])
def test_fused_rope_equals_rope_then_attention(wbits, hd, neox):
    """Un-rotated q / k_new with the tables == rope_ followed by the plain call, bit for bit, cache bytes included; at
    positions past 32 k, in the passes regime (32 heads over 8, B = 9)."""
    from exllamav2_b200 import ext as ext_c
    H, KVH, B = 32, 8, 9
    cap = alp.largest_fit(wbits, hd, H, B) + ar.PAGE
    c, q, kn, vn = small_case(wbits, hd, H, KVH, B, cap, [cap - 1 - 1000 * b for b in range(B)], seed=hd + wbits)
    sin_np, cos_np = oracle.rope_tables(hd, cap)
    sin, cos = torch.from_numpy(sin_np).to(DEV), torch.from_numpy(cos_np).to(DEV)
    sl = torch.from_numpy(np.array(c["seqlens"], dtype=np.int32)).to(DEV)
    qt, kt = torch.from_numpy(q).to(DEV), torch.from_numpy(kn).to(DEV)
    fused_cache = device_cache(c)
    o1 = launch(c, qt, kt, vn, fused_cache, rope=(sin, cos, 2 if neox else 1))
    qr, kr = qt.clone().view(B, 1, H * hd), kt.clone().view(B, 1, KVH * hd)
    ext_c.rope_(qr, sin, cos, -1, H, hd, sl, neox)
    ext_c.rope_(kr, sin, cos, -1, KVH, hd, sl, neox)
    plain_cache = device_cache(c)
    o2 = launch(c, qr.view(B, 1, H, hd), kr.view(B, 1, KVH, hd), vn, plain_cache)
    for a, b in zip(fused_cache, plain_cache):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))
    assert torch.equal(o1.view(torch.int16), o2.view(torch.int16))


@pytest.mark.parametrize("wbits,hd", [(4, 128), (6, 64), (8, 128)])
def test_captured_launch_replays_eager_bits(wbits, hd):
    """A launch of the passes regime captured in a CUDA graph (64 heads, B = 1, split) replays to the eager bits."""
    from exllamav2_b200 import ext as ext_c
    H, KVH, B = 64, 8, 1
    cap = 131072 if hd == 128 else 262144
    c, q, kn, vn = small_case(wbits, hd, H, KVH, B, cap, [cap - 5000], seed=3)
    assert alp.long_plan(wbits, hd, H, B, 1, cap)["passes"]
    cache = device_cache(c)
    qt, kt, vt = (torch.from_numpy(a).to(DEV) for a in (q, kn, vn))
    s = torch.cuda.Stream(DEV)
    out_g = torch.zeros(q.shape, dtype=torch.half, device=DEV)
    with torch.cuda.stream(s):
        launch(c, qt, kt, vt, cache, out=out_g)             # the first launch on s creates its split scratch, uncaptured
    eager = out_g.clone()
    out_g.fill_(0)
    sl, bt = torch.tensor(c["seqlens"], dtype=torch.int32, device=DEV), torch.from_numpy(c["bt"]).to(DEV)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        ext_c.paged_attn_decode_q4(qt, kt, vt, *cache, sl, bt, out_g, c["sigma"], wbits=wbits)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out_g.view(torch.int16), eager.view(torch.int16))
    compare(eager.cpu().numpy(), truth(c, q, kn, vn), ("graph", wbits, hd, "random"))


# ---- the page-table refusal ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("wbits,hd", FMTS)
def test_largest_page_table_runs_and_one_more_is_refused(wbits, hd):
    """The largest page table a single-token launch accepts (attn_long_plan: the table plus a pass of 512 positions fill
    200 KB) runs a 1000-position sequence correctly; one page more raises an error naming the pages and the bytes and
    writes nothing.  Only the pages the sequence uses exist."""
    from exllamav2_b200 import ext as ext_c
    H, KVH = 8, 8
    most = alp.largest_page_table(wbits, hd)
    for pps, ok in ((most, True), (most + 1, False)):
        c, q, kn, vn = small_case(wbits, hd, H, KVH, 1, 4 * ar.PAGE, [1000], seed=pps)
        bt = np.zeros((1, pps), np.int32)
        bt[0, :4] = c["bt"][0]
        c["bt"] = bt
        lp = alp.long_plan(wbits, hd, H, 1, 1, pps * ar.PAGE)
        assert lp["passes"] and lp["fits"] == ok and lp["pass_len"] == alp.PASS_MIN
        cache = device_cache(c)
        if ok:
            compare(launch(c, q, kn, vn, cache).cpu().numpy(), truth(c, q, kn, vn), ("largest_table", wbits, hd, "random"))
            continue
        before = [a.clone() for a in cache]
        out = torch.full(q.shape, 3.0, dtype=torch.half, device=DEV)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
        with pytest.raises(RuntimeError, match=f"page table of {pps} pages needs {lp['smem']} bytes"):
            ext_c.paged_attn_decode_q4(t(q), t(kn), t(vn), *cache, t(np.array([1000], np.int32)), t(bt), out, c["sigma"],
                                       wbits=wbits)
        torch.cuda.synchronize()
        assert all(torch.equal(a.view(torch.uint8), b.view(torch.uint8)) for a, b in zip(before, cache))
        assert (out == 3.0).all()


def test_report_errors():
    """Prints the worst errors of the cases above that ran (DESIGN.md §3.4 quotes them)."""
    for k in sorted(MEASURED, key=str):
        print("worst", k, "rel-L2 %.2e  elem %.2e" % MEASURED[k])
