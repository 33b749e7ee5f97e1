"""Fused K/V-cache decode attention (csrc/attn_q4.cu) in every regime its host launches, for Q4 / Q6 / Q8 at head dims 64
and 128, against fp64 softmax attention over the oracle-dequantised cache plus the unquantised new rows.

The regimes, and the branch tests/attn_regimes.py's plan() asserts each one lands in (sequence lengths come from the plan):
  global_qlen   q_len 4 over a 4096-position cache: no split, cached rows past the staged window read from global memory
  global_q1     q_len 1 over a 1024-position cache (too short to split), seqlen in (stage, 1023]
  ring          16384 positions, q_len 1: the streaming ring under split-KV, B = 2 (one full sequence, one ragged)
  ring_qlen     12288 positions, q_len 2 / 4 / 8: no split, one CTA streams the whole cache once per query; the new rows sit
                inside the last sub-chunk, exactly at a sub-chunk start, and across a page end
  split_batch   B = 4, GQA, 4096 positions: lengths 0, 1, 1500 (ragged last chunk) and 4095 (full) in one launch
  split_batch3  B = 3: lengths 511 (one chunk: no merge), 2047, 1025
  batched       H = 32, KVH = 8, B = 8 / 9, 4096 positions: no split, more CTAs than SMs, one CTA over up to 4095 positions

Inputs (`mode`):
  random  q ~ N(0, 4), new rows ~ N(0, 1) over a cache of random bytes
  needle  q and the keys are built in the stored (rotated) domain so that a few positions per head (every boundary the
          plan names, dealt round robin over the heads: 2-8 per head, up to ~40 at 16 k with 16 chunks; and every appended row) carry all but ~1e-13 of the softmax mass, 40 nats above the background with
          score gaps of 0.25 nat; each needle's value row is a one-hot in its own 32-value block, whose scale differs from its
          neighbours'.  A mis-addressed needle moves the output by O(1/8).
  zero    q = 0: every position gets the same weight, so the output is the mean of every value row, each counted once
  sink / deep / sink_last (split_batch only): a needle 6 nats above the rest in the first chunk, a whole chunk 100 nats
          below the rest (its merge weight underflows), and the new row as the sink in the last chunk
Every case checks the cache bytes (the appended rows are this library's fp16_to_q_kv, at Q4 also the oracle's; nothing else
moved), the output against fp64 per (b, i, h), and that a second launch gives the same bits.

Tolerances (TOL below) were set from the errors measured on an H100 80GB HBM3, see TOL.
"""
import functools
import zlib

import numpy as np
import pytest
import torch

import attn_regimes as ar
import cases
import exl2_oracle as oracle

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FMTS = [(w, hd) for w in (4, 6, 8) for hd in (64, 128)]
S0 = 40.0          # needle score above a zero score, nats
BETA = 16.0        # needle query amplitude (a power of two: the rotated query is exact)
MEASURED = {}      # (branch, wbits, hd, mode) -> (rel-L2, max abs err / max |truth|), the worst case of the run

# Per-(b, i, h) limits: rel-L2, and the largest element error relative to max |truth|.  Worst cases measured over every
# test of this file on an H100 80GB HBM3 (DESIGN.md §3.4 has them per branch): rel-L2 8.5e-4 (batched, random inputs),
# element 1.5e-3 (split_batch, skewed merge).  Most of it is the truth's own fp16 rounding: the oracle dequantises the
# cache as the reference does, through fp16 Hadamard sums, while the kernel forms scores and P V from the stored integers in
# fp32.  The limits sit ~1.7-1.9x above the worst measured values.
TOL = dict(rel=1.6e-3, mx=2.5e-3)


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def regime(name, wbits, hd):
    st = ar.smem_bytes(wbits, hd, 1, 4096, 1)["stage"]
    rst, sub = ar.smem_bytes(wbits, hd, 2, 12288, 1)["stage"], ar.smem_bytes(wbits, hd, 2, 12288, 1)["sub"]
    if name == "global_qlen":
        return dict(H=8, KVH=2, q_len=4, max_ctx=4096, seqlens=[st - 1, st + 1, 4092], expect={"global"})
    if name == "global_q1":
        return dict(H=8, KVH=8, q_len=1, max_ctx=1024, seqlens=[st + 1, 1023], expect={"global"})
    if name == "ring":
        return dict(H=8, KVH=8, q_len=1, max_ctx=16384, seqlens=[16383, 9000], expect={"ring", "merge_batch"})
    if name == "ring_qlen":
        q_len = {4: 4, 6: 8, 8: 2}[wbits]
        return dict(H=8, KVH=8, q_len=q_len, max_ctx=12288, seqlens=[rst + 40 * sub + 37, rst + 60 * sub, 40 * 256 - q_len // 2],
                    expect={"ring_qlen"})
    if name == "split_batch":
        return dict(H=8, KVH=2, q_len=1, max_ctx=4096, seqlens=[0, 1, 1500, 4095], expect={"merge_batch"})
    if name == "split_batch3":
        return dict(H=8, KVH=8, q_len=1, max_ctx=4096, seqlens=[511, 2047, 1025], expect={"merge_batch"})
    if name == "batched":
        sl = [0, 1, 255, 256, 511, 512, 513, 4095] + ([3000] if hd == 128 else [])
        return dict(H=32, KVH=8, q_len=1, max_ctx=4096, seqlens=sl, expect={"batched", "global"})
    # the 70B preset's heads (H 64, KVH 8): 264 / 64 = 4 chunks at B = 1, and at B = 8 more CTAs than SMs without split
    if name == "heads64_q1":
        return dict(H=64, KVH=8, q_len=1, max_ctx=4096, seqlens=[4095], expect={"merge", "global"}, nsplit=4)
    if name == "heads64_ring":
        return dict(H=64, KVH=8, q_len=1, max_ctx=16384, seqlens=[16383], expect={"merge", "ring"}, nsplit=4)
    if name == "heads64_batched":
        return dict(H=64, KVH=8, q_len=1, max_ctx=4096, seqlens=[0, 1, 255, 256, 513, 1500, 3000, 4095],
                    expect={"batched", "global"}, nsplit=1)
    # a GQA ratio that is not a power of two (Qwen2.5-7B: 28 heads over 4 kv heads): 264 / 28 = 9 chunks of 512 positions
    if name == "gqa7_split9":
        return dict(H=28, KVH=4, q_len=1, max_ctx=4608, seqlens=[4607], expect={"merge"}, nsplit=9)
    raise KeyError(name)


REGIMES = ["global_qlen", "global_q1", "ring", "ring_qlen", "split_batch", "split_batch3", "batched"]
WIDE = ["heads64_q1", "heads64_ring", "heads64_batched", "gqa7_split9"]      # hd 128 only, the head dim of the models they stand for


def ek_of(h, group, hd):
    """Stored coordinate of head h's key direction (distinct among the heads sharing a kv head)."""
    return ((h % group) * 37 + 3) % hd


def cv_of(j, h, hd):
    """Stored coordinate of needle j's value one-hot (distinct for j < 8, in different 32-value blocks)."""
    return (j * (hd // 8) + 3 * h) % hd


def key_scale(score, sigma, beta, bits):
    return ar.round8(score / (sigma * beta * ar.one_hot_amp(bits)))


def stable_seed(*key):
    return zlib.crc32(repr(key).encode())


@functools.lru_cache(maxsize=1)
def base_case(wbits, hd, name, sigma_key=None, beta=BETA):
    """Block table, cache bytes (random background + the needle rows) and the needle map of one regime; shared by its modes."""
    r = regime(name, wbits, hd)
    H, KVH, q_len, max_ctx, seqlens = r["H"], r["KVH"], r["q_len"], r["max_ctx"], r["seqlens"]
    B, pps, group = len(seqlens), max_ctx // ar.PAGE, H // KVH
    kb, vb = ar.widths(wbits)
    p = ar.plan(wbits, hd, H, B, q_len, max_ctx, seqlens)
    got = ar.branches(p, q_len, H, B)
    assert r["expect"] <= got, (name, r["expect"], got)
    assert p["nsplit"] == r.get("nsplit", p["nsplit"]), (name, p["nsplit"])
    sigma = sigma_key if sigma_key is not None else 1.0 / np.sqrt(hd)
    rng = np.random.default_rng(stable_seed(wbits, hd, name))
    pages_total = B * pps + 1                      # one page no sequence owns: nothing may write it
    bt = rng.permutation(pages_total)[:B * pps].reshape(B, pps).astype(np.int32)
    shp = (pages_total, ar.PAGE, KVH)
    kq = rng.integers(0, 256, size=shp + (hd * kb // 8,), dtype=np.uint8)
    vq = rng.integers(0, 256, size=shp + (hd * vb // 8,), dtype=np.uint8)
    ks = (rng.uniform(0.05, 0.15, size=shp + (hd // 32,)) / (16 if kb == 8 else 1)).astype(np.float16)
    vs = (rng.uniform(0.02, 0.3, size=shp + (hd // 32,)) / (16 if vb == 8 else 1)).astype(np.float16)
    # needles: each boundary position of sequence b goes to one head (round robin); its row at that head's kv head becomes a
    # one-hot key at the head's coordinate with a designed scale, and a one-hot value in its own block
    needles = []                                   # (b, pos, h, slot)
    for b in range(B):
        per_head = {}
        for k, pos in enumerate(ar.boundary_positions(p, b)):
            h = (k + b) % H
            j = per_head.setdefault(h, 0)
            per_head[h] = j + 1
            pg, rr, g = bt[b, pos // ar.PAGE], pos % ar.PAGE, h // group
            kq[pg, rr, g] = ar.s_one_hot_row(hd, kb, ek_of(h, group, hd))
            ks[pg, rr, g, ek_of(h, group, hd) // 32] = key_scale(S0 + 0.25 * (j % 8), sigma, beta, kb)
            cv = cv_of(j % 8, h, hd)
            vq[pg, rr, g] = ar.s_one_hot_row(hd, vb, cv)
            vs[pg, rr, g, cv // 32] = ar.round8(rng.uniform(0.5, 1.0) * 8 / ar.one_hot_amp(vb))
            needles.append((b, pos, h, j))
    return dict(r=r, plan=p, H=H, KVH=KVH, q_len=q_len, max_ctx=max_ctx, seqlens=seqlens, B=B, group=group, sigma=sigma, beta=beta,
                bt=bt, kq=kq, ks=ks, vq=vq, vs=vs, needles=needles, kb=kb, vb=vb)


def _rows(c, kq, ks, vq, vs):
    K = [ar.gather_rows(kq, ks, c["bt"], b, sl, c["kb"]) for b, sl in enumerate(c["seqlens"])]
    V = [ar.gather_rows(vq, vs, c["bt"], b, sl, c["vb"]) for b, sl in enumerate(c["seqlens"])]
    return K, V


@functools.lru_cache(maxsize=1)
def base_rows(wbits, hd, name, sigma_key=None, beta=BETA):
    c = base_case(wbits, hd, name, sigma_key, beta)
    return _rows(c, c["kq"], c["ks"], c["vq"], c["vs"])


def make_inputs(c, mode, rng, hd, sink_new=None, shave=0):
    """q, k_new, v_new.  needle: head h's query is beta * (the sign pattern of its key direction), less 2^-11 on `shave` of
    its elements, so its rotated block holds (32 - shave * 2^-11) * beta on one coordinate and zeros elsewhere."""
    B, q_len, H, KVH, group, sigma, beta = c["B"], c["q_len"], c["H"], c["KVH"], c["group"], c["sigma"], c["beta"]
    kn = rng.normal(0, 1, size=(B, q_len, KVH, hd)).astype(np.float16)
    vn = rng.normal(0, 1, size=(B, q_len, KVH, hd)).astype(np.float16)
    if mode == "random":
        return rng.normal(0, 4, size=(B, q_len, H, hd)).astype(np.float16), kn, vn
    if mode == "zero":
        return np.zeros((B, q_len, H, hd), np.float16), kn, vn
    q = np.zeros((B, q_len, H, hd), np.float16)
    kn[:] = 0
    for h in range(H):
        d = ar.key_direction(hd, c["kb"], ek_of(h, group, hd))
        sg = np.sign(d)
        sg[np.nonzero(sg)[0][:shave]] *= 1 - 2.0 ** -11
        q[:, :, h] = (beta * sg).astype(np.float16)
        nj = {b: sum(1 for (bb, _, hh, _) in c["needles"] if bb == b and hh == h) for b in range(B)}
        for b in range(B):
            for i in range(q_len):             # every appended row is a needle of every head
                sc = S0 + 0.25 * ((nj[b] + i) % 8)
                if sink_new is not None and i == q_len - 1:
                    sc = sink_new
                s = key_scale(sc, sigma, beta, c["kb"])
                kn[b, i, h // group] = (kn[b, i, h // group].astype(np.float64) + d * float(s)).astype(np.float16)
    return q, kn, vn


def launch(c, q, kn, vn, kq, ks, vq, vs, out_consumer=0, sigma=None):
    from exllamav2_b200 import ext as ext_c
    gk, gks, gv, gvs = t(kq), t(ks), t(vq), t(vs)
    out = torch.zeros(q.shape, dtype=torch.half, device=DEV)
    ext_c.paged_attn_decode_q4(t(q), t(kn), t(vn), gk, gks, gv, gvs, t(np.array(c["seqlens"], dtype=np.int32)), t(c["bt"]), out,
                               c["sigma"] if sigma is None else sigma, out_consumer, wbits={(4, 4): 4, (8, 4): 6, (8, 8): 8}[(c["kb"], c["vb"])])
    torch.cuda.synchronize()
    assert ext_c.paged_attn_status(DEV) == 0
    return out.cpu().numpy(), gk.cpu().numpy(), gks.cpu().numpy(), gv.cpu().numpy(), gvs.cpu().numpy()


def check_cache(c, kn, vn, kq0, ks0, vq0, vs0, kq1, ks1, vq1, vs1, wbits):
    """The appended rows are bit-exact with this library's fp16_to_q_kv (and at Q4 with the oracle); nothing else moved."""
    from exllamav2_b200 import ext as ext_c
    B, q_len, KVH = c["B"], c["q_len"], c["KVH"]
    hd = kn.shape[-1]
    # all appended rows as one token of a whole number of 512-value blocks (zero rows after them), so the non-paged pack
    # converts exactly these rows and widens nothing
    n = B * q_len * KVH
    npad = -(-n * hd // 512) * 512 // hd
    def pad(x):
        z = torch.zeros((1, 1, npad, hd), dtype=torch.half, device=DEV)
        z.view(npad, hd)[:n] = t(x).view(n, hd)
        return z
    kt, vt = pad(kn), pad(vn)
    pk = torch.zeros((1, 1, npad, hd * c["kb"] // 8), dtype=torch.uint8, device=DEV)
    pv = torch.zeros((1, 1, npad, hd * c["vb"] // 8), dtype=torch.uint8, device=DEV)
    pks = torch.zeros((1, 1, npad, hd // 32), dtype=torch.half, device=DEV)
    pvs = torch.zeros_like(pks)
    ext_c.fp16_to_q_kv(kt, pk, pks, vt, pv, pvs, 1, 0, 1, 0, ext_c.none_tensor, ext_c.none_tensor, wbits)
    torch.cuda.synchronize()
    shp = lambda a: a.cpu().numpy().reshape(npad, -1)[:n].reshape(B, q_len, KVH, -1)
    pk, pks, pv, pvs = shp(pk), shp(pks), shp(pv), shp(pvs)
    if wbits == 4:
        ok_, oks = oracle.kv_pack_q4(kn)
        ov_, ovs = oracle.kv_pack_q4(vn)
        assert np.array_equal(pk, ok_) and np.array_equal(pv, ov_)
        assert np.array_equal(cases.u16(pks), cases.u16(oks)) and np.array_equal(cases.u16(pvs), cases.u16(ovs))
    want = [a.copy() for a in (kq0, ks0, vq0, vs0)]
    for b, sl in enumerate(c["seqlens"]):
        for i in range(q_len):
            pg, rr = c["bt"][b, (sl + i) // ar.PAGE], (sl + i) % ar.PAGE
            want[0][pg, rr], want[1][pg, rr], want[2][pg, rr], want[3][pg, rr] = pk[b, i], pks[b, i], pv[b, i], pvs[b, i]
    assert np.array_equal(kq1, want[0]) and np.array_equal(vq1, want[2])
    assert np.array_equal(cases.u16(ks1), cases.u16(want[1])) and np.array_equal(cases.u16(vs1), cases.u16(want[3]))


def compare(got, truth, tag, tol=TOL):
    B, q_len, H, hd = truth.shape
    g = got.astype(np.float64)
    assert np.isfinite(g).all(), tag
    d = np.linalg.norm(g - truth, axis=-1)
    n = np.linalg.norm(truth, axis=-1)
    rel = d / np.where(n > 0, n, 1.0)
    mx = np.abs(g - truth).max(-1) / np.maximum(np.abs(truth).max(-1), 1e-30)
    worst = (float(rel.max()), float(mx.max()))
    old = MEASURED.get(tag, (0.0, 0.0))
    MEASURED[tag] = (max(old[0], worst[0]), max(old[1], worst[1]))
    bad = np.argwhere((rel > tol["rel"]) | (mx > tol["mx"]))
    assert len(bad) == 0, (tag, [(tuple(x), rel[tuple(x)], mx[tuple(x)]) for x in bad[:8]])


def run_case(c, wbits, hd, q, kn, vn, kq, ks, vq, vs, K, V, tag, sigma=None):
    out, kq1, ks1, vq1, vs1 = launch(c, q, kn, vn, kq, ks, vq, vs, sigma=sigma)
    check_cache(c, kn, vn, kq, ks, vq, vs, kq1, ks1, vq1, vs1, wbits)
    truth, probs = ar.attention_truth(q, kn, vn, K, V, c["seqlens"], c["sigma"] if sigma is None else sigma, return_probs=True)
    compare(out, truth, tag)
    out2 = launch(c, q, kn, vn, kq, ks, vq, vs, sigma=sigma)[0]
    assert np.array_equal(out.view(np.uint16), out2.view(np.uint16)), "a second identical launch gave different bits"
    return out, truth, probs


def needle_mask(c, b, h, extra=()):
    """Positions of sequence b that are needles of head h (cached needles, the sink rows, every appended row)."""
    sl = c["seqlens"][b]
    m = np.zeros(sl + c["q_len"], dtype=bool)
    for (bb, pos, hh, _) in c["needles"]:
        if bb == b and hh == h:
            m[pos] = True
    for (bb, pos, hh) in extra:
        if bb == b and hh == h:
            m[pos] = True
    m[sl:] = True
    return m


CASES = [(w, hd, name, mode) for (w, hd) in FMTS for name in REGIMES + WIDE for mode in ("random", "needle", "zero")
         if hd == 128 or name not in WIDE]


@pytest.mark.parametrize("wbits,hd,name,mode", CASES)
def test_regime(wbits, hd, name, mode):
    c = base_case(wbits, hd, name)
    K, V = base_rows(wbits, hd, name)
    rng = np.random.default_rng(stable_seed(wbits, hd, name, mode))
    q, kn, vn = make_inputs(c, mode, rng, hd)
    out, truth, probs = run_case(c, wbits, hd, q, kn, vn, c["kq"], c["ks"], c["vq"], c["vs"], K, V, (name, wbits, hd, mode))
    if mode == "zero":            # every position counted once: the mean of all value rows (causal for the new rows)
        for b, sl in enumerate(c["seqlens"]):
            for i in range(c["q_len"]):
                Vb = np.concatenate([V[b], vn[b, :i + 1].astype(np.float64)], 0)
                mean = Vb.mean(0)                                       # [KVH, hd]
                assert np.allclose(truth[b, i], np.repeat(mean, c["group"], 0), rtol=1e-9, atol=1e-12)
    if mode == "needle":          # the design: needles carry all but ~1e-9 of every head's mass
        for b in range(c["B"]):
            for h in range(c["H"]):
                m = needle_mask(c, b, h)
                assert (probs[b][:, h][:, m].sum(-1) > 1 - 1e-9).all(), (b, h)


def deep_row(hd, bits, es):
    """Stored values all zero except -8 at each coordinate in es: every head of the group scores it far below."""
    if bits == 8:
        row = np.full(hd, 128, dtype=np.uint8)
        row[es] = 120
        return row
    row = np.full(hd // 2, 0x88, dtype=np.uint8)
    for e in es:
        row[e // 2] &= 0xF0 if e % 2 == 0 else 0x0F
    return row


def _chunks(c, b):
    return [(x["p_lo"], x["p_hi"]) for x in c["plan"]["ctas"] if x["b"] == b]


SKEW_CASES = [(w, hd, "split_batch") for (w, hd) in FMTS] + [(w, 128, n) for w in (4, 6, 8) for n in ("heads64_q1", "gqa7_split9")]


@pytest.mark.parametrize("wbits,hd,name", SKEW_CASES)
@pytest.mark.parametrize("skew", ["sink", "deep", "sink_last"])
def test_skewed_merge(wbits, hd, name, skew):
    """Split-KV whose chunks' maxima differ widely.  sink: a needle 6 nats above the rest in the first chunk of every split
    sequence, the other chunks still carrying 1-10 % of the mass, so a merge that drops their rescale or weight fails.
    deep: the second chunk's rows all score ~100 nats below the rest; its merge weight underflows to zero and the output
    stays finite.  sink_last: the sink is the appended row, in the last chunk.  Added needles skip positions that already hold
    one (the plan's boundary needles), which with 64 heads fall inside the range they are spread over."""
    c0 = base_case(wbits, hd, name)
    c = dict(c0)
    kq, ks, vq, vs = (c0[k].copy() for k in ("kq", "ks", "vq", "vs"))
    H, group, kb, sigma = c["H"], c["group"], c["kb"], c["sigma"]
    split = [b for b in range(c["B"]) if len(_chunks(c, b)) >= 3]
    assert split
    extra = []
    taken = {(n[0], n[1]) for n in c0["needles"]}

    def free(b, pos):
        while (b, pos) in taken:
            pos += 1
        taken.add((b, pos))
        return pos

    if skew in ("sink", "sink_last"):
        # three more needles of every head at S0 in each chunk the sink is not in: together they carry a few % of the mass
        for b in split:
            ch = _chunks(c, b)
            for lo, hi in (ch[1:] if skew == "sink" else ch[:-1]):
                for h in range(H):
                    for k in range(3):
                        pos = free(b, lo + 20 + 4 * h + k)
                        pg, rr, g = c["bt"][b, pos // ar.PAGE], pos % ar.PAGE, h // group
                        kq[pg, rr, g] = ar.s_one_hot_row(hd, kb, ek_of(h, group, hd))
                        ks[pg, rr, g, ek_of(h, group, hd) // 32] = key_scale(S0, sigma, c["beta"], kb)
                        extra.append((b, pos, h))
    if skew == "sink":
        for b in split:
            lo, hi = _chunks(c, b)[0]
            for h in range(H):
                pos = free(b, lo + 100 + 3 * h)                     # inside the first chunk, no boundary
                pg, rr, g = c["bt"][b, pos // ar.PAGE], pos % ar.PAGE, h // group
                kq[pg, rr, g] = ar.s_one_hot_row(hd, kb, ek_of(h, group, hd))
                ks[pg, rr, g, ek_of(h, group, hd) // 32] = key_scale(S0 + 6.0, sigma, c["beta"], kb)
                extra.append((b, pos, h))
    if skew == "deep":
        c["needles"] = [n for n in c0["needles"] if not (n[0] in split and _chunks(c, n[0])[1][0] <= n[1] < _chunks(c, n[0])[1][1])]
        for b in split:
            lo, hi = _chunks(c, b)[1]
            for pos in range(lo, hi):
                pg, rr = c["bt"][b, pos // ar.PAGE], pos % ar.PAGE
                for g in range(c["KVH"]):
                    kq[pg, rr, g] = deep_row(hd, kb, [ek_of(h, group, hd) for h in range(group)])
                    ks[pg, rr, g] = ar.round8(60.0 / (sigma * c["beta"] * 8))
    K, V = _rows(c, kq, ks, vq, vs)
    rng = np.random.default_rng(stable_seed(wbits, hd, skew))
    q, kn, vn = make_inputs(c, "needle", rng, hd, sink_new=(S0 + 6.0) if skew == "sink_last" else None)
    out, truth, probs = run_case(c, wbits, hd, q, kn, vn, kq, ks, vq, vs, K, V, (name, wbits, hd, skew))
    for b in split:
        ch = _chunks(c, b)
        for h in range(H):
            pr = probs[b][0, h]
            assert pr[needle_mask(c, b, h, extra)].sum() > 1 - 1e-9
            if skew == "sink":
                rest = 1 - pr[ch[0][0]:ch[0][1]].sum()
                assert 0.01 <= rest <= 0.10, (b, h, rest)
            if skew == "sink_last":
                rest = 1 - pr[ch[-1][0]:ch[-1][1]].sum()
                assert 0.01 <= rest <= 0.10, (b, h, rest)
            if skew == "deep":
                s = np.log(pr[ch[1][0]:ch[1][1]].max() + 1e-300) - np.log(pr.max())
                assert s < -95, (b, h, s)


# ---- the query's power-of-two guard -------------------------------------------------------------------------------------

L2E = np.float32(1.4426950408889634)           # the kernel's log2(e) (attn_q4.cu exl2b_paged_attn_decode_q, P.scale_log2)


def _edge_query(target, hd, kb):
    """(softmax_scale, shave) that put the needle query's rotated block maximum (beta = 1) exactly on `target`, found by
    running the kernel's fp32 rotation (attn_regimes.rotate_q_fp32) over nearby fp32 scales and shaved queries."""
    f32 = np.float32
    d = ar.key_direction(hd, kb, ek_of(0, 1, hd))
    for shave in range(16):
        sg = np.sign(d)
        sg[np.nonzero(sg)[0][:shave]] *= 1 - 2.0 ** -11
        qrow = sg.astype(np.float16)
        base = f32(target / ((32 - shave * 2.0 ** -11) / 32.0) / float(L2E))
        up = dn = base
        for _ in range(300):
            for s in (up, dn):
                if np.abs(ar.rotate_q_fp32(qrow, f32(s * L2E)).reshape(-1, 32)).max() == f32(target):
                    return float(s), shave
            up, dn = np.nextafter(up, f32(np.inf), dtype=f32), np.nextafter(dn, f32(-np.inf), dtype=f32)
    raise AssertionError("no fp32 softmax_scale reaches the target")


# block maxima: on a power of two; the largest the guard bumps to the next exponent (2 - 2^-14 of the binade); the next one
# below, which is quantised to 32767 under the lower exponent; and the largest fp32 below the power of two
EDGES = {"pow2": 4.0, "guard_bumped": 2.0 * (2 - 2.0 ** -14), "below_guard": 2.0 * (2 - 2.0 ** -14 - 2.0 ** -23),
         "just_below": 2.0 * (2 - 2.0 ** -23)}


EDGE_CASES = [(w, hd, "global_q1") for (w, hd) in FMTS] + [(w, 128, n) for w in (4, 6, 8) for n in ("heads64_q1", "gqa7_split9")]


@pytest.mark.parametrize("wbits,hd,name", EDGE_CASES)
@pytest.mark.parametrize("edge", list(EDGES))
def test_query_block_max_at_power_of_two(wbits, hd, name, edge):
    """rotate_q quantises each rotated 32-value query block to 16 bits under a power-of-two scale chosen from
    amax * 1.000030518, so the largest value stays inside the signed high byte.  The needle query's block maximum is put
    exactly on a power of two, just below it, and on both sides of that guard; the host's fp32 rotation confirms where it
    lands, and the needles' weights must still be read back within the usual tolerance."""
    kb, _ = ar.widths(wbits)
    sigma, shave = _edge_query(EDGES[edge], hd, kb)
    c = base_case(wbits, hd, name, sigma_key=sigma, beta=1.0)
    K, V = base_rows(wbits, hd, name, sigma_key=sigma, beta=1.0)
    rng = np.random.default_rng(5)
    q, kn, vn = make_inputs(c, "needle", rng, hd, shave=shave)
    scale_log2 = np.float32(np.float32(sigma) * L2E)
    for h in range(c["H"]):
        amax = np.abs(ar.rotate_q_fp32(q[0, 0, h], scale_log2)).max()
        assert amax == np.float32(EDGES[edge]), (h, amax, EDGES[edge])
    bumped = np.float32(amax * np.float32(1.000030518)) >= 2.0 ** (np.floor(np.log2(amax)) + 1)
    assert bumped == (edge in ("guard_bumped", "just_below"))
    run_case(c, wbits, hd, q, kn, vn, c["kq"], c["ks"], c["vq"], c["vs"], K, V, (name, wbits, hd, "edge_" + edge), sigma=sigma)


# ---- the chained output, read by its consumer ---------------------------------------------------------------------------

CHAIN = [  # (B, q_len, max_ctx, seqlens, merge)
    (1, 1, 4096, [3000], True), (2, 1, 4096, [3000, 1100], True), (5, 1, 4096, [4095, 1025, 2000, 600, 3500], True),
    (8, 1, 4096, [1100 + 300 * i for i in range(8)], True),
    (1, 1, 1024, [700], False), (1, 2, 2048, [1500], False), (1, 5, 4096, [600], False), (1, 8, 4096, [3000], False),
]


@pytest.mark.parametrize("wbits", [4, 6, 8])
@pytest.mark.parametrize("B,q_len,max_ctx,seqlens,merge", CHAIN)
def test_chained_output_read_by_o_proj(wbits, B, q_len, max_ctx, seqlens, merge):
    """With out_consumer = o_proj the kernel leaves its output in o_proj's activation buffer: a plain fp16 row in o_proj's
    stored-row order for one row, the core-matrix operand layout for 2-8 rows; from the single-CTA branch and from the merge.
    o_proj run on that buffer must equal, bit for bit, o_proj run on the plain output, since the consumer sees the same fp16
    values.  One row is read by the single-row integer GEMV, whose prepared-row entry point (gemv_norm, prepared=True)
    applies RMSNorm, so both sides take that entry point with a unit weight; gemm_half_q_half_prepared reads the core-matrix
    layout at every row count and is the consumer for 2-8 rows only."""
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200 import synthetic
    from exllamav2_b200.linear import ExLlamaV2Linear
    H, KVH, hd = 8, 2, 128
    p = ar.plan(wbits, hd, H, B, q_len, max_ctx, seqlens)
    assert ("merge" in ar.branches(p, q_len, H, B)) == merge
    kb, vb = ar.widths(wbits)
    rng = np.random.default_rng(B * 10 + q_len)
    pps = max_ctx // ar.PAGE
    bt = rng.permutation(B * pps).reshape(B, pps).astype(np.int32)
    shp = (B * pps, ar.PAGE, KVH)
    kq = rng.integers(0, 256, size=shp + (hd * kb // 8,), dtype=np.uint8)
    vq = rng.integers(0, 256, size=shp + (hd * vb // 8,), dtype=np.uint8)
    ks = (rng.uniform(0.05, 0.15, size=shp + (hd // 32,)) / (16 if kb == 8 else 1)).astype(np.float16)
    vs = (rng.uniform(0.02, 0.3, size=shp + (hd // 32,)) / (16 if vb == 8 else 1)).astype(np.float16)
    lin = ExLlamaV2Linear(H * hd, 512, device=DEV)
    lin.load(synthetic.random_linear(H * hd, 512, ((4,), (1.0,), 128), device=DEV, seed=4))
    q = rng.normal(0, 4, size=(B, q_len, H, hd)).astype(np.float16)
    kn = rng.normal(0, 1, size=(B, q_len, KVH, hd)).astype(np.float16)
    vn = rng.normal(0, 1, size=(B, q_len, KVH, hd)).astype(np.float16)
    c = dict(seqlens=seqlens, bt=bt, sigma=1.0 / np.sqrt(hd), kb=kb, vb=vb)
    out, *_ = launch(c, q, kn, vn, kq, ks, vq, vs, out_consumer=lin.q_handle)
    rows = B * q_len
    y_chain = torch.zeros((rows, 512), dtype=torch.half, device=DEV)
    y_plain = torch.zeros((rows, 512), dtype=torch.half, device=DEV)
    x = t(out).view(rows, H * hd)
    if rows == 1:
        # one row is left as a plain fp16 row in o_proj's stored-row order, which the single-row integer GEMV reads; its
        # entry point for a prepared row applies RMSNorm, so both sides go through the same norm (unit weight)
        w = torch.ones(H * hd, dtype=torch.half, device=DEV)
        ext_c.gemv_norm(x, lin.q_handle, w, 1e-6, y_chain, prepared=True)
        ext_c.gemv_norm(x, lin.q_handle, w, 1e-6, y_plain)
    else:
        ext_c.gemm_half_q_half_prepared(lin.q_handle, y_chain, False, 0.0)
        ext_c.gemm_half_q_half(x, lin.q_handle, y_plain)
    torch.cuda.synchronize()
    assert torch.equal(y_chain.view(torch.int16), y_plain.view(torch.int16)), \
        oracle.rel_l2(y_chain.float().cpu().numpy(), y_plain.float().cpu().numpy())
    # and the attention output the consumer read is right
    K = [ar.gather_rows(kq, ks, bt, b, sl, kb) for b, sl in enumerate(seqlens)]
    V = [ar.gather_rows(vq, vs, bt, b, sl, vb) for b, sl in enumerate(seqlens)]
    compare(out, ar.attention_truth(q, kn, vn, K, V, seqlens, c["sigma"]), ("chain", wbits, hd, f"{B}x{q_len}"))
    lin.unload()


# ---- the shared-memory refusal ------------------------------------------------------------------------------------------

def _largest_fit(wbits, hd, q_len):
    pages = 1
    while ar.smem_bytes(wbits, hd, q_len, (pages + 1) * ar.PAGE, 1)["fits"]:
        pages += 1
    return pages * ar.PAGE


@pytest.mark.parametrize("wbits", [4, 6, 8])
def test_largest_context_runs_and_one_page_more_is_refused(wbits):
    """q_len 2 (no split): the score buffer holds the whole cache.  At the largest cache whose shared memory fits (plan():
    28928 positions at Q4, 29696 at Q8) the full sequence runs through the ring and matches fp64; one page more raises an
    error naming the context and writes nothing."""
    from exllamav2_b200 import ext as ext_c
    hd, H, KVH, q_len = 128, 2, 2, 2
    kb, vb = ar.widths(wbits)
    ctx = _largest_fit(wbits, hd, q_len)
    rng = np.random.default_rng(wbits)
    for pps, ok in ((ctx // ar.PAGE, True), (ctx // ar.PAGE + 1, False)):
        bt = rng.permutation(pps).reshape(1, pps).astype(np.int32)
        shp = (pps, ar.PAGE, KVH)
        kq = rng.integers(0, 256, size=shp + (hd * kb // 8,), dtype=np.uint8)
        vq = rng.integers(0, 256, size=shp + (hd * vb // 8,), dtype=np.uint8)
        ks = (rng.uniform(0.05, 0.15, size=shp + (hd // 32,)) / (16 if kb == 8 else 1)).astype(np.float16)
        vs = (rng.uniform(0.02, 0.3, size=shp + (hd // 32,)) / (16 if vb == 8 else 1)).astype(np.float16)
        seqlens = [pps * ar.PAGE - q_len]
        q = rng.normal(0, 4, size=(1, q_len, H, hd)).astype(np.float16)
        kn = rng.normal(0, 1, size=(1, q_len, KVH, hd)).astype(np.float16)
        vn = rng.normal(0, 1, size=(1, q_len, KVH, hd)).astype(np.float16)
        c = dict(seqlens=seqlens, bt=bt, sigma=1.0 / np.sqrt(hd), kb=kb, vb=vb, B=1, q_len=q_len, KVH=KVH)
        if ok:
            assert "ring_qlen" in ar.branches(ar.plan(wbits, hd, H, 1, q_len, pps * ar.PAGE, seqlens), q_len, H, 1)
            K = [ar.gather_rows(kq, ks, bt, 0, seqlens[0], kb)]
            V = [ar.gather_rows(vq, vs, bt, 0, seqlens[0], vb)]
            run_case(c, wbits, hd, q, kn, vn, kq, ks, vq, vs, K, V, ("largest", wbits, hd, "random"))
            continue
        assert not ar.smem_bytes(wbits, hd, q_len, pps * ar.PAGE, 1)["fits"]
        gk, gks, gv, gvs = t(kq), t(ks), t(vq), t(vs)
        out = torch.full((1, q_len, H, hd), 3.0, dtype=torch.half, device=DEV)
        with pytest.raises(RuntimeError, match=f"context of {pps * ar.PAGE} tokens"):
            ext_c.paged_attn_decode_q4(t(q), t(kn), t(vn), gk, gks, gv, gvs, t(np.array(seqlens, dtype=np.int32)), t(bt), out,
                                       c["sigma"], wbits=wbits)
        torch.cuda.synchronize()
        assert np.array_equal(gk.cpu().numpy(), kq) and np.array_equal(gv.cpu().numpy(), vq)
        assert np.array_equal(cases.u16(gks.cpu().numpy()), cases.u16(ks)) and np.array_equal(cases.u16(gvs.cpu().numpy()), cases.u16(vs))
        assert (out == 3.0).all()
