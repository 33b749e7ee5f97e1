"""The Q6 and Q8 K/V caches on the GPU: fp16_to_q_kv / q_to_fp16_kv with wbits 6 and 8, decode attention straight over the
8-bit keys (and values), the decoder with cache_bits 6 / 8, and the reference's own ExLlamaV2Cache_Q6 / _Q8 on the drop-in.

  * pack / unpack vs the reference extension's outputs (tests/golden/ref_kv_q68.npz, bit-exact) and vs the oracle
    (tests/kv_q68.py, bytes within +-1 where the reciprocal-based division rounds differently);
  * fused attention: the appended rows' cache bytes are the oracle's pack and nothing else moved; the output is within
    2e-3 rel-L2 of fp64 softmax attention over the oracle-dequantised cache plus the unquantised new rows;
  * split-KV, the streaming ring, fused RoPE, the page guard and the chained output on 8-bit caches;
  * on the same K / V the attention error orders Q8 < Q6 < Q4 (a kernel that drops bits fails this).
"""
import os
import sys
import types

import numpy as np
import pytest
import torch

import cases
import exl2_oracle as oracle
import kv_q68

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_kv_q68.npz")
PYPKG = os.path.join(ROOT, "oracle", "_ref", "pypkg")
# Logit tolerances (rel-L2) of the decoder tests, from the measured runs (2 layers, 4 decode steps, H100):
#   test-small, fused vs ref and chained vs fused: Q6 <= 6.6e-3, Q8 <= 2.8e-3;  test-tiny chained vs fused: Q6 5.5e-3, Q8 2.7e-3
#   test-tiny, fused vs ref: Q8 6.0e-3; Q6 4e-2 to 9.8e-2.  There the reference re-quantises neighbouring tokens on every append
#   (a 128-wide kv row is a quarter of a 512-value block, cache.cu:177-184) and the fused kernel quantises each row once; Q6's
#   4-bit values drift the most, so at Q6 (as at Q4, test_gpu_decoder.py) test-tiny compares only the two fused sequences.
# Q4's LOGIT_TOL is 5e-2 (test_gpu_decoder.py).
LOGIT_TOL = {6: 1.5e-2, 8: 1e-2}
TINY_REF_TOL = {8: 1.5e-2}


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _state(x_shape, bits, fill=0):
    shp = tuple(x_shape[:-1])
    return (torch.full(shp + (x_shape[-1] * bits // 8,), fill, dtype=torch.uint8, device=DEV),
            torch.full(shp + (x_shape[-1] // 32,), float(fill), dtype=torch.half, device=DEV))


def _off_by_one_ok(got_q, want_q, bits):
    def el(q):
        q = np.asarray(q, dtype=np.uint8)
        if bits == 8:
            return q.astype(np.int32)
        return np.stack([q & 15, q >> 4], -1).astype(np.int32)
    d = el(got_q) - el(want_q)
    return np.abs(d).max() <= 1 and np.count_nonzero(d) <= 2e-3 * d.size


# ---- pack / unpack ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("wbits", [6, 8])
@pytest.mark.parametrize("name", list(kv_q68.NONPAGED))
def test_kv_nonpaged_vs_reference(name, wbits):
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200.ext import none_tensor
    gold = np.load(GOLDEN)
    c = kv_q68.NONPAGED[name]
    kb, vb = kv_q68.widths(wbits)
    k, v = kv_q68.nonpaged_inputs(name)
    kq, ks = _state(k.shape, kb)
    vq, vs = _state(v.shape, vb)
    B = c["shape"][0]
    ext_c.fp16_to_q_kv(t(k), kq, ks, t(v), vq, vs, B, c["offset"], c["width"], 0, none_tensor, none_tensor, wbits)
    ko, vo = torch.zeros_like(t(k)), torch.zeros_like(t(v))
    ext_c.q_to_fp16_kv(kq, ko, ks, vq, vo, vs, B, c["offset"], c["width"], 0, none_tensor, none_tensor, wbits)
    torch.cuda.synchronize()
    tag = f"{name}_w{wbits}_"
    a, b = kv_q68.nonpaged_range(name)
    for x, item, q, s, o, bits in ((k, "k", kq, ks, ko, kb), (v, "v", vq, vs, vo, vb)):
        gq, gs = q.cpu().numpy(), s.cpu().numpy().view(np.uint16)
        assert np.array_equal(gq, gold[tag + item + "q"]) and np.array_equal(gs, gold[tag + item + "s"]), "pack differs from the reference"
        assert np.array_equal(kv_q68.digest(o.cpu().numpy()), gold[tag + item + "o"]), "unpack differs from the reference"
        pq, ps = kv_q68.kv_pack(x[:, a:b].reshape(B, b - a, -1), bits)
        assert np.array_equal(gs.reshape(B, x.shape[1], -1)[:, a:b], ps.view(np.uint16))
        assert _off_by_one_ok(gq.reshape(B, x.shape[1], -1)[:, a:b], pq, bits)


@pytest.mark.parametrize("wbits", [6, 8])
@pytest.mark.parametrize("name", list(kv_q68.PAGED))
def test_kv_paged_vs_reference(name, wbits):
    from exllamav2_b200 import ext as ext_c
    gold = np.load(GOLDEN)
    c = kv_q68.PAGED[name]
    kb, vb = kv_q68.widths(wbits)
    k, v = kv_q68.paged_inputs(name)
    kq, ks = _state(k.shape, kb)
    vq, vs = _state(v.shape, vb)
    bt, sl = t(np.array(c["block_table"], dtype=np.int32)), t(np.array(c["seqlens"], dtype=np.int32))
    kt, vt = t(k), t(v)
    ext_c.fp16_to_q_kv(kt, kq, ks, vt, vq, vs, 2, 0, c["q_len"], kv_q68.PAGE, sl, bt, wbits)
    ko, vo = torch.zeros_like(kt), torch.zeros_like(vt)
    ext_c.q_to_fp16_kv(kq, ko, ks, vq, vo, vs, 2, 0, 0, kv_q68.PAGE, sl + c["q_len"], bt, wbits)
    torch.cuda.synchronize()
    tag = f"{name}_w{wbits}_"
    rows = kv_q68.paged_rows(name)
    pg, rr = np.array([r[2] for r in rows]), np.array([r[3] for r in rows])
    for x, item, q, s, o, bits in ((k, "k", kq, ks, ko, kb), (v, "v", vq, vs, vo, vb)):
        gq, gs = q.cpu().numpy(), s.cpu().numpy().view(np.uint16)
        for a, it in ((gq, "q"), (gs, "s")):
            assert np.array_equal(kv_q68.digest(a), gold[tag + item + it]), f"{item}{it} differs from the reference"
        assert np.array_equal(kv_q68.digest(o.cpu().numpy()), gold[tag + item + "o"]), "unpack differs from the reference"
        pq, ps = kv_q68.kv_pack(x[pg, rr], bits)
        assert np.array_equal(gs[pg, rr], ps.view(np.uint16)) and _off_by_one_ok(gq[pg, rr], pq, bits)


@pytest.mark.parametrize("wbits", [6, 8])
def test_kv_partial_range_leaves_rest_untouched(wbits):
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200.ext import none_tensor
    kb, vb = kv_q68.widths(wbits)
    B, S, H, D = 2, 12, 8, 128
    k = torch.randn((B, S, H, D), dtype=torch.half, device=DEV)
    v = torch.randn((B, S, H, D), dtype=torch.half, device=DEV)
    kq, ks = _state(k.shape, kb, 0xAB)
    vq, vs = _state(v.shape, vb, 0xAB)
    ks.fill_(7.0)
    vs.fill_(7.0)
    ext_c.fp16_to_q_kv(k, kq, ks, v, vq, vs, B, 5, 3, 0, none_tensor, none_tensor, wbits)
    torch.cuda.synchronize()
    for q, s in ((kq, ks), (vq, vs)):
        assert (q[:, :5] == 0xAB).all() and (q[:, 8:] == 0xAB).all() and (s[:, :5] == 7.0).all() and (s[:, 8:] == 7.0).all()
        assert not (q[:, 5:8] == 0xAB).all() and not (s[:, 5:8] == 7.0).all()


@pytest.mark.parametrize("wbits", [4, 6, 8])
def test_kv_widening_stays_inside_the_tensor(wbits):
    """A row of 2 * 64 values is a quarter of a 512-value block, so one token widens to four.  With one token per batch row
    the widening must stop at the end of each row: every row is converted as itself, and the memory after the last row (two
    guard rows of the same allocation here) is neither read into nor written.  A range outside the rows is refused."""
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200.ext import none_tensor
    kb, vb = kv_q68.widths(wbits)
    R = 6
    big = torch.randn((R + 2, 1, 2, 64), dtype=torch.half, device=DEV)
    kq, ks = _state(big.shape, kb, 0xAB)
    vq, vs = _state(big.shape, vb, 0xAB)
    ks.fill_(7.0)
    vs.fill_(7.0)
    ext_c.fp16_to_q_kv(big[:R], kq[:R], ks[:R], big[:R], vq[:R], vs[:R], R, 0, 1, 0, none_tensor, none_tensor, wbits)
    torch.cuda.synchronize()
    x = big[:R].cpu().numpy()
    for q, s, bits in ((kq, ks, kb), (vq, vs, vb)):
        assert (q[R:] == 0xAB).all() and (s[R:] == 7.0).all(), "wrote past the last row"
        pq, ps = kv_q68.kv_pack(x.reshape(R, 1, -1), bits)
        assert np.array_equal(cases.u16(s[:R].cpu().numpy().reshape(R, 1, -1)), cases.u16(ps))
        assert _off_by_one_ok(q[:R].cpu().numpy().reshape(R, 1, -1), pq, bits)
    out = torch.full((R + 2, 1, 2, 64), 3.0, dtype=torch.half, device=DEV)
    out_v = out.clone()
    ext_c.q_to_fp16_kv(kq[:R], out[:R], ks[:R], vq[:R], out_v[:R], vs[:R], R, 0, 1, 0, none_tensor, none_tensor, wbits)
    torch.cuda.synchronize()
    for o, q, s, bits in ((out, kq, ks, kb), (out_v, vq, vs, vb)):
        assert (o[R:] == 3.0).all(), "wrote past the last row"
        want = kv_q68.kv_unpack(q[:R].cpu().numpy().reshape(R, 1, -1), s[:R].cpu().numpy().reshape(R, 1, -1), bits)
        assert np.array_equal(cases.u16(o[:R].cpu().numpy().reshape(R, 1, -1)), cases.u16(want))
    with pytest.raises(RuntimeError, match="outside the tensor"):
        ext_c.fp16_to_q_kv(big[:R], kq[:R], ks[:R], big[:R], vq[:R], vs[:R], R, 0, 2, 0, none_tensor, none_tensor, wbits)
    with pytest.raises(RuntimeError, match="outside the tensor"):
        ext_c.fp16_to_q_kv(big[:R], kq[:R], ks[:R], big[:R], vq[:R], vs[:R], R + 1, 0, 1, 0, none_tensor, none_tensor, wbits)


def test_kv_rejects_bad_wbits_and_shapes():
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200.ext import none_tensor
    k = torch.randn((1, 4, 8, 64), dtype=torch.half, device=DEV)
    q4, s = _state(k.shape, 4)
    q8, _ = _state(k.shape, 8)
    with pytest.raises(RuntimeError, match=r"wbits must be 4 \(Q4\), 6 \(Q6\) or 8 \(Q8\); got 5"):
        ext_c.fp16_to_q_kv(k, q8, s, k, q8.clone(), s.clone(), 1, 0, 4, 0, none_tensor, none_tensor, 5)
    with pytest.raises(RuntimeError, match="key states have last dimension 32"):          # Q8 keys need 64 bytes per row
        ext_c.fp16_to_q_kv(k, q4, s, k, q8, s.clone(), 1, 0, 4, 0, none_tensor, none_tensor, 8)
    with pytest.raises(RuntimeError, match="value states have last dimension 64"):        # Q6 values are 4-bit
        ext_c.q_to_fp16_kv(q8, k.clone(), s, q8.clone(), k.clone(), s.clone(), 1, 0, 4, 0, none_tensor, none_tensor, 6)
    with pytest.raises(RuntimeError, match="key states have last dimension 64"):          # Q4 keys are 4-bit
        ext_c.fp16_to_q_kv(k, q8, s, k, q4, s.clone(), 1, 0, 4, 0, none_tensor, none_tensor, 4)


# ---- fused attention -------------------------------------------------------------------------------------------------

def _paged_cache(rng, pages_total, page, KVH, hd, wbits):
    kb, vb = kv_q68.widths(wbits)
    past_k = rng.normal(0, 1, size=(pages_total, page, KVH, hd)).astype(np.float16)
    past_v = rng.normal(0, 1, size=(pages_total, page, KVH, hd)).astype(np.float16)
    kq0, ks0 = kv_q68.kv_pack(past_k, kb)
    vq0, vs0 = kv_q68.kv_pack(past_v, vb)
    return kq0, ks0, vq0, vs0


def _attn_truth(q, kn, vn, K_deq, V_deq, block_table, seqlens, page, b, i, h, group, hd):
    rows = [(block_table[b, p // page], p % page) for p in range(seqlens[b])]
    K = np.stack([K_deq[pg, r, h // group] for pg, r in rows] + [kn[b, j, h // group].astype(np.float64) for j in range(i + 1)])
    V = np.stack([V_deq[pg, r, h // group] for pg, r in rows] + [vn[b, j, h // group].astype(np.float64) for j in range(i + 1)])
    s = K @ q[b, i, h].astype(np.float64) / np.sqrt(hd)
    pr = np.exp(s - s.max())
    return (pr / pr.sum()) @ V


@pytest.mark.parametrize("wbits", [6, 8])
@pytest.mark.parametrize("H,KVH,hd,q_len,seqlens", [
    (8, 8, 128, 1, [300, 0]),          # crosses a page; an empty sequence
    (8, 2, 64, 3, [17, 255]),          # GQA, several new rows, append runs over a page end
    (4, 4, 128, 8, [511, 5]),
])
def test_paged_attn_decode_q68(H, KVH, hd, q_len, seqlens, wbits):
    from exllamav2_b200 import ext as ext_c
    kb, vb = kv_q68.widths(wbits)
    page, pps = 256, 3
    B = len(seqlens)
    rng = np.random.default_rng(31)
    pages_total = B * pps + 1
    block_table = rng.permutation(pages_total)[:B * pps].reshape(B, pps).astype(np.int32)
    kq0, ks0, vq0, vs0 = _paged_cache(rng, pages_total, page, KVH, hd, wbits)
    q = rng.normal(0, 1, size=(B, q_len, H, hd)).astype(np.float16)
    kn = rng.normal(0, 1, size=(B, q_len, KVH, hd)).astype(np.float16)
    vn = rng.normal(0, 1, size=(B, q_len, KVH, hd)).astype(np.float16)
    kq, ks, vq, vs = t(kq0), t(ks0), t(vq0), t(vs0)
    out = torch.zeros((B, q_len, H, hd), dtype=torch.half, device=DEV)
    ext_c.paged_attn_decode_q4(t(q), t(kn), t(vn), kq, ks, vq, vs, t(np.array(seqlens, dtype=np.int32)), t(block_table), out,
                               1.0 / np.sqrt(hd), wbits=wbits)
    torch.cuda.synchronize()
    kq1, ks1, vq1, vs1 = kq.cpu().numpy(), ks.cpu().numpy(), vq.cpu().numpy(), vs.cpu().numpy()
    got = out.cpu().numpy()
    # 1. the appended rows are exactly what fp16_to_q_kv stores (the kernel divides like the GPU pack); nothing else moved
    want_kq, want_ks, want_vq, want_vs = kq0.copy(), ks0.copy(), vq0.copy(), vs0.copy()
    nkq, nks = kv_q68.kv_pack(kn, kb)
    nvq, nvs = kv_q68.kv_pack(vn, vb)
    for b in range(B):
        for i in range(q_len):
            pos = seqlens[b] + i
            pg = block_table[b, pos // page]
            want_kq[pg, pos % page], want_ks[pg, pos % page] = nkq[b, i], nks[b, i]
            want_vq[pg, pos % page], want_vs[pg, pos % page] = nvq[b, i], nvs[b, i]
    assert np.array_equal(cases.u16(ks1), cases.u16(want_ks)) and np.array_equal(cases.u16(vs1), cases.u16(want_vs))
    assert _off_by_one_ok(kq1, want_kq, kb) and _off_by_one_ok(vq1, want_vq, vb)
    # ... and bit-exactly what this library's fp16_to_q_kv stores for the same rows
    kt, vt = t(kn).view(B * q_len, 1, KVH, hd), t(vn).view(B * q_len, 1, KVH, hd)
    pk, pks = _state(kt.shape, kb)
    pv, pvs = _state(vt.shape, vb)
    ext_c.fp16_to_q_kv(kt, pk, pks, vt, pv, pvs, B * q_len, 0, 1, 0, ext_c.none_tensor, ext_c.none_tensor, wbits)
    torch.cuda.synchronize()
    pk, pv = pk.cpu().numpy().reshape(B, q_len, KVH, -1), pv.cpu().numpy().reshape(B, q_len, KVH, -1)
    for b in range(B):
        for i in range(q_len):
            pos = seqlens[b] + i
            pg = block_table[b, pos // page]
            assert np.array_equal(kq1[pg, pos % page], pk[b, i]) and np.array_equal(vq1[pg, pos % page], pv[b, i])
            want_kq[pg, pos % page], want_vq[pg, pos % page] = pk[b, i], pv[b, i]
    assert np.array_equal(kq1, want_kq) and np.array_equal(vq1, want_vq)
    # 2. attention over the dequantised cache
    kd = kv_q68.kv_unpack(kq1, ks1, kb).astype(np.float64)
    vd = kv_q68.kv_unpack(vq1, vs1, vb).astype(np.float64)
    group = H // KVH
    for b in range(B):
        for i in range(q_len):
            for h in range(H):
                ref = _attn_truth(q, kn, vn, kd, vd, block_table, seqlens, page, b, i, h, group, hd)
                err = oracle.rel_l2(got[b, i, h].astype(np.float64), ref)
                assert err < 2e-3, (b, i, h, err)


def _long_setup(H, KVH, hd, pps, B, seed, wbits):
    page = 256
    rng = np.random.default_rng(seed)
    pages_total = B * pps
    block_table = rng.permutation(pages_total).reshape(B, pps).astype(np.int32)
    kq0, ks0, vq0, vs0 = _paged_cache(rng, pages_total, page, KVH, hd, wbits)
    return page, rng, block_table, kq0, ks0, vq0, vs0


@pytest.mark.parametrize("H,KVH,hd,ctx,cache_len", [
    (32, 32, 128, 1000, 1024 * 2),      # split-KV, 2 chunks
    (32, 8, 128, 4095, 4096),           # GQA, 8 chunks, ragged last chunk
    (8, 8, 64, 16000, 16384),           # the streaming ring (cache > 8192 positions)
    (32, 32, 128, 9000, 12288),         # ring + split-KV at hd 128
    (32, 32, 128, 130, 16384),          # short context in a long cache: one active chunk
])
def test_q8_long_context(H, KVH, hd, ctx, cache_len):
    from exllamav2_b200 import ext as ext_c
    wbits = 8
    page, rng, block_table, kq0, ks0, vq0, vs0 = _long_setup(H, KVH, hd, cache_len // 256, 1, ctx, wbits)
    q = rng.normal(0, 1, size=(1, 1, H, hd)).astype(np.float16)
    kn = rng.normal(0, 1, size=(1, 1, KVH, hd)).astype(np.float16)
    vn = rng.normal(0, 1, size=(1, 1, KVH, hd)).astype(np.float16)
    kq, ks, vq, vs = t(kq0), t(ks0), t(vq0), t(vs0)
    out = torch.zeros((1, 1, H, hd), dtype=torch.half, device=DEV)
    sl = t(np.array([ctx], dtype=np.int32))
    pg = block_table[0, np.arange(ctx) // page]
    r = np.arange(ctx) % page
    K = np.concatenate([kv_q68.kv_unpack_q8(kq0[pg, r], ks0[pg, r]).astype(np.float64), kn[0].astype(np.float64)], axis=0)
    V = np.concatenate([kv_q68.kv_unpack_q8(vq0[pg, r], vs0[pg, r]).astype(np.float64), vn[0].astype(np.float64)], axis=0)
    group = H // KVH
    for rep in range(2):          # twice: the merge counters must be back at zero after a launch
        kq.copy_(t(kq0)); ks.copy_(t(ks0)); vq.copy_(t(vq0)); vs.copy_(t(vs0))
        ext_c.paged_attn_decode_q4(t(q), t(kn), t(vn), kq, ks, vq, vs, sl, t(block_table), out, 1.0 / np.sqrt(hd), wbits=wbits)
        torch.cuda.synchronize()
        assert ext_c.paged_attn_status(DEV) == 0
        got = out[0, 0].cpu().numpy().astype(np.float64)
        for h in range(H):
            s = K[:, h // group] @ q[0, 0, h].astype(np.float64) / np.sqrt(hd)
            pr = np.exp(s - s.max())
            err = oracle.rel_l2(got[h], (pr / pr.sum()) @ V[:, h // group])
            assert err < 2e-3, (rep, h, err)
    nkq, _ = kv_q68.kv_pack_q8(kn)
    pgn = block_table[0, ctx // page]
    assert _off_by_one_ok(kq.cpu().numpy()[pgn, ctx % page], nkq[0, 0], 8)


@pytest.mark.parametrize("wbits", [6, 8])
@pytest.mark.parametrize("H,KVH,hd,neox", [(32, 32, 128, True), (32, 4, 64, True), (8, 8, 128, False), (8, 2, 64, False)])
def test_q68_fused_rope_equals_rope_then_attention(H, KVH, hd, neox, wbits):
    from exllamav2_b200 import ext as ext_c
    page, rng, block_table, kq0, ks0, vq0, vs0 = _long_setup(H, KVH, hd, 2, 2, 7, wbits)
    B = 2
    seqlens = np.array([77, 300], dtype=np.int32)
    sin_np, cos_np = oracle.rope_tables(hd, 512)
    sin, cos = t(sin_np), t(cos_np)
    q = t(rng.normal(0, 1, size=(B, 1, H, hd)).astype(np.float16))
    kn = t(rng.normal(0, 1, size=(B, 1, KVH, hd)).astype(np.float16))
    vn = t(rng.normal(0, 1, size=(B, 1, KVH, hd)).astype(np.float16))
    sl, bt = t(seqlens), t(block_table)

    def run(fused):
        kq, ks, vq, vs = t(kq0), t(ks0), t(vq0), t(vs0)
        out = torch.zeros((B, 1, H, hd), dtype=torch.half, device=DEV)
        if fused:
            ext_c.paged_attn_decode_q4(q, kn, vn, kq, ks, vq, vs, sl, bt, out, 1.0 / np.sqrt(hd), rope=(sin, cos, 2 if neox else 1),
                                       wbits=wbits)
        else:
            qr, kr = q.clone().view(B, 1, H * hd), kn.clone().view(B, 1, KVH * hd)
            ext_c.rope_(qr, sin, cos, -1, H, hd, sl, neox)
            ext_c.rope_(kr, sin, cos, -1, KVH, hd, sl, neox)
            ext_c.paged_attn_decode_q4(qr.view(B, 1, H, hd), kr.view(B, 1, KVH, hd), vn, kq, ks, vq, vs, sl, bt, out, 1.0 / np.sqrt(hd),
                                       wbits=wbits)
        torch.cuda.synchronize()
        return out, kq, ks
    o1, kq1, ks1 = run(True)
    o2, kq2, ks2 = run(False)
    assert torch.equal(kq1, kq2) and torch.equal(ks1.view(torch.int16), ks2.view(torch.int16))
    assert torch.equal(o1.view(torch.int16), o2.view(torch.int16))


@pytest.mark.parametrize("wbits", [6, 8])
def test_q68_page_table_overrun_is_refused(wbits):
    from exllamav2_b200 import ext as ext_c
    H = KVH = 4
    hd = 64
    page, rng, block_table, kq0, ks0, vq0, vs0 = _long_setup(H, KVH, hd, 1, 1, 3, wbits)
    q = t(rng.normal(0, 1, size=(1, 2, H, hd)).astype(np.float16))
    kn = t(rng.normal(0, 1, size=(1, 2, KVH, hd)).astype(np.float16))
    vn = t(rng.normal(0, 1, size=(1, 2, KVH, hd)).astype(np.float16))
    kq, ks, vq, vs = t(kq0), t(ks0), t(vq0), t(vs0)
    out = torch.zeros((1, 2, H, hd), dtype=torch.half, device=DEV)
    ext_c.paged_attn_clear_status(DEV)
    ext_c.paged_attn_decode_q4(q, kn, vn, kq, ks, vq, vs, t(np.array([255], dtype=np.int32)), t(block_table), out, 0.125, wbits=wbits)
    torch.cuda.synchronize()
    assert ext_c.paged_attn_status(DEV) & 1
    assert torch.equal(kq, t(kq0)) and torch.equal(vq, t(vq0)) and torch.count_nonzero(out).item() == 0
    ext_c.paged_attn_clear_status(DEV)
    assert ext_c.paged_attn_status(DEV) == 0


@pytest.mark.parametrize("wbits", [4, 6, 8])
@pytest.mark.parametrize("B,q_len", [(1, 1), (2, 3)])
def test_chained_output_leaves_plain_output_unchanged(wbits, B, q_len):
    """With out_consumer (o_proj) the kernel also writes the consumer's activation buffer; the plain output is the same bits."""
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200 import synthetic
    from exllamav2_b200.linear import ExLlamaV2Linear
    H, KVH, hd = 8, 2, 128
    page, rng, block_table, kq0, ks0, vq0, vs0 = _long_setup(H, KVH, hd, 2, B, 9, wbits)
    lin = ExLlamaV2Linear(H * hd, 512, device=DEV)
    lin.load(synthetic.random_linear(H * hd, 512, ((4,), (1.0,), 128), device=DEV, seed=4))
    q = t(rng.normal(0, 1, size=(B, q_len, H, hd)).astype(np.float16))
    kn = t(rng.normal(0, 1, size=(B, q_len, KVH, hd)).astype(np.float16))
    vn = t(rng.normal(0, 1, size=(B, q_len, KVH, hd)).astype(np.float16))
    sl, bt = t(np.array([100, 311][:B], dtype=np.int32)), t(block_table)
    outs = []
    for oc in (0, lin.q_handle):
        kq, ks, vq, vs = t(kq0), t(ks0), t(vq0), t(vs0)
        out = torch.zeros((B, q_len, H, hd), dtype=torch.half, device=DEV)
        ext_c.paged_attn_decode_q4(q, kn, vn, kq, ks, vq, vs, sl, bt, out, 1.0 / np.sqrt(hd), oc, wbits=wbits)
        torch.cuda.synchronize()
        outs.append((out, kq, vq))
    assert torch.equal(outs[0][0].view(torch.int16), outs[1][0].view(torch.int16))
    assert torch.equal(outs[0][1], outs[1][1]) and torch.equal(outs[0][2], outs[1][2])
    lin.unload()


def test_error_orders_q8_q6_q4():
    """The same unquantised K / V stored as Q4, Q6 and Q8: the attention output's error against fp64 attention over the
    UNQUANTISED rows must shrink with every added bit (measured: Q4 0.20, Q6 0.10, Q8 1.1e-2 rel-L2)."""
    from exllamav2_b200 import ext as ext_c
    H, KVH, hd, ctx = 8, 8, 128, 700
    page = 256
    rng = np.random.default_rng(17)
    block_table = np.arange(3, dtype=np.int32).reshape(1, 3)
    past_k = rng.normal(0, 1, size=(3, page, KVH, hd)).astype(np.float16)
    past_v = rng.normal(0, 1, size=(3, page, KVH, hd)).astype(np.float16)
    q = rng.normal(0, 1, size=(1, 1, H, hd)).astype(np.float16) * np.float16(2.0)
    kn = rng.normal(0, 1, size=(1, 1, KVH, hd)).astype(np.float16)
    vn = rng.normal(0, 1, size=(1, 1, KVH, hd)).astype(np.float16)
    K = np.concatenate([past_k.reshape(-1, KVH, hd)[:ctx], kn[0]], 0).astype(np.float64)
    V = np.concatenate([past_v.reshape(-1, KVH, hd)[:ctx], vn[0]], 0).astype(np.float64)
    truth = np.stack([(lambda s: (np.exp(s - s.max()) / np.exp(s - s.max()).sum()) @ V[:, h])(K[:, h] @ q[0, 0, h].astype(np.float64) / np.sqrt(hd))
                      for h in range(H)])
    errs = {}
    for wbits in (4, 6, 8):
        kb, vb = kv_q68.widths(wbits)
        kq, ks = (t(a) for a in kv_q68.kv_pack(past_k, kb))
        vq, vs = (t(a) for a in kv_q68.kv_pack(past_v, vb))
        out = torch.zeros((1, 1, H, hd), dtype=torch.half, device=DEV)
        ext_c.paged_attn_decode_q4(t(q), t(kn), t(vn), kq, ks, vq, vs, t(np.array([ctx], dtype=np.int32)), t(block_table), out,
                                   1.0 / np.sqrt(hd), wbits=wbits)
        torch.cuda.synchronize()
        errs[wbits] = oracle.rel_l2(out[0, 0].cpu().numpy().astype(np.float64), truth)
    assert errs[8] < errs[6] < errs[4], errs
    assert errs[8] < errs[4] / 4, errs


# ---- decoder ---------------------------------------------------------------------------------------------------------

def _run(mode, preset, prompt, gen_ids, graph, cache_bits):
    from exllamav2_b200.model import ExLlamaV2Decoder, PRESETS
    dec = ExLlamaV2Decoder(PRESETS[preset](), device=DEV, seed=3, batch_size=prompt.shape[0], cache_len=512, cache_bits=cache_bits)
    assert dec.cache.wbits == cache_bits
    dec.fused_attn = mode != "ref"
    dec.chained = mode == "chained"
    dec.prefill(prompt)
    if graph:
        dec.capture()
    outs = [dec.decode(gen_ids[:, i:i + 1]).float().cpu().numpy().copy() for i in range(gen_ids.shape[1])]
    kq = dec.cache.key_states[0].cpu().numpy().copy()
    dec.unload()
    return outs, kq


@pytest.mark.parametrize("cache_bits", [6, 8])
@pytest.mark.parametrize("preset", ["test-small", "test-tiny"])
def test_decoder_sequences_agree(preset, cache_bits):
    g = torch.Generator().manual_seed(5)
    prompt = torch.randint(0, 512, (1, 11), generator=g).to(DEV)
    gen = torch.randint(0, 512, (1, 4), generator=g).to(DEV)
    ref, kq_ref = _run("ref", preset, prompt, gen, False, cache_bits)
    fus, kq_fus = _run("fused", preset, prompt, gen, False, cache_bits)
    chn, _ = _run("chained", preset, prompt, gen, False, cache_bits)
    for i in range(gen.shape[1]):
        assert np.isfinite(chn[i]).all()
        e1, e2 = oracle.rel_l2(fus[i], ref[i]), oracle.rel_l2(chn[i], fus[i])
        if preset == "test-small" or cache_bits == 8:
            assert e1 < (TINY_REF_TOL if preset == "test-tiny" else LOGIT_TOL)[cache_bits], (i, e1)
        assert e2 < LOGIT_TOL[cache_bits], (i, e2)
    if preset == "test-small":       # a 512-value kv row: the reference's block-wise re-quantisation touches no neighbour
        assert np.array_equal(kq_ref, kq_fus)


@pytest.mark.parametrize("cache_bits", [6, 8])
def test_decoder_graph_matches_eager(cache_bits):
    g = torch.Generator().manual_seed(6)
    prompt = torch.randint(0, 512, (1, 7), generator=g).to(DEV)
    gen = torch.randint(0, 512, (1, 5), generator=g).to(DEV)
    eager, _ = _run("chained", "test-tiny", prompt, gen, False, cache_bits)
    graph, _ = _run("chained", "test-tiny", prompt, gen, True, cache_bits)
    for a, b in zip(eager, graph):
        assert np.array_equal(a, b)


def test_decoder_rejects_unknown_cache_bits():
    from exllamav2_b200.model import ExLlamaV2Decoder, PRESETS
    with pytest.raises(ValueError, match="cache_bits must be 4"):
        ExLlamaV2Decoder(PRESETS["test-tiny"](), device=DEV, cache_len=512, cache_bits=5)


# ---- drop-in: the reference's own ExLlamaV2Cache_Q6 / _Q8 ---------------------------------------------------------------

@pytest.fixture(scope="module")
def ref_py():
    if not os.path.exists(os.path.join(PYPKG, "exllamav2", "__init__.pyc")):
        pytest.skip("oracle/_ref/pypkg not built (python oracle/build_ref.py)")
    import exllamav2_b200.ext as b200_ext
    b200_ext.install_as_exllamav2_ext()
    sys.path.insert(0, PYPKG)
    import exllamav2                                  # noqa: F401  the reference package, unmodified
    from exllamav2 import ext as ref_ext
    assert ref_ext.ext_c is b200_ext, "the reference did not pick up the drop-in module"
    return types.SimpleNamespace(ext=ref_ext, b200=b200_ext)


def _stub_model(kvh, hd, layers):
    """What ExLlamaV2Cache_Q reads from its model (cache.py:30-75, 420-460): config, cache_map, get_cache_devices()."""
    cfg = types.SimpleNamespace(max_seq_len=512, num_key_value_heads=kvh, num_hidden_layers=layers, head_dim=hd,
                                max_batch_size=1, max_input_len=512)
    return types.SimpleNamespace(config=cfg, cache_map={i: DEV for i in range(layers)}, get_cache_devices=lambda: [DEV],
                                 tp_context=None)


@pytest.mark.parametrize("cls", ["ExLlamaV2Cache_Q6", "ExLlamaV2Cache_Q8"])
def test_reference_cache_on_dropin(ref_py, cls):
    import exllamav2.cache as ref_cache
    kvh, hd = 8, 64
    cache = getattr(ref_cache, cls)(_stub_model(kvh, hd, 2), batch_size=1, max_seq_len=512)
    kb, vb = kv_q68.widths(cache.wbits)
    assert cache.key_states[0].shape[-1] == hd * kb // 8 and cache.value_states[0].shape[-1] == hd * vb // 8
    rng = np.random.default_rng(2)
    tk, tv = cache.temp_tensors[DEV]
    k = rng.normal(0, 1, size=tuple(tk.shape)).astype(np.float16)
    v = rng.normal(0, 1, size=tuple(tv.shape)).astype(np.float16)
    # non-paged: tokens [3, 9) of layer 1
    tk.copy_(t(k)); tv.copy_(t(v))
    cache.store_kv_state(1, 1, 3, 6)
    torch.cuda.synchronize()
    for st, ss, x, bits in ((cache.key_states[1], cache.key_scales[1], k, kb), (cache.value_states[1], cache.value_scales[1], v, vb)):
        pq, ps = kv_q68.kv_pack(x[:, 3:9].reshape(1, 6, -1), bits)
        got_q, got_s = st[:, 3:9].cpu().numpy().reshape(1, 6, -1), ss[:, 3:9].cpu().numpy().reshape(1, 6, -1)
        assert np.array_equal(cases.u16(got_s), cases.u16(ps)) and _off_by_one_ok(got_q, pq, bits)
        assert not st[:, :3].any() and not st[:, 9:].any()
    tk.zero_(); tv.zero_()
    ok, ov = cache.get_kv_state(1, 1, 3, 6)
    torch.cuda.synchronize()
    want_k = kv_q68.kv_unpack(cache.key_states[1][:, 3:9].cpu().numpy(), cache.key_scales[1][:, 3:9].cpu().numpy(), kb)
    want_v = kv_q68.kv_unpack(cache.value_states[1][:, 3:9].cpu().numpy(), cache.value_scales[1][:, 3:9].cpu().numpy(), vb)
    assert np.array_equal(cases.u16(ok[:, 3:9].cpu().numpy()), cases.u16(want_k))
    assert np.array_equal(cases.u16(ov[:, 3:9].cpu().numpy()), cases.u16(want_v))
    # paged: the cache's 512 positions as two pages of 256, the second first; append 4 tokens at position 254 (crosses a page)
    bt = torch.tensor([[1, 0]], dtype=torch.int32, device=DEV)
    sl = torch.tensor([254], dtype=torch.int32, device=DEV)
    for L in (cache.key_states[0], cache.value_states[0], cache.key_scales[0], cache.value_scales[0]):
        L.zero_()
    tk.copy_(t(k)); tv.copy_(t(v))
    cache.store_kv_state(0, 1, 0, 4, page_size=256, cache_seqlens=sl, block_table=bt)
    torch.cuda.synchronize()
    kp = cache.key_states[0].view(2, 256, kvh, -1).cpu().numpy()
    kps = cache.key_scales[0].view(2, 256, kvh, -1).cpu().numpy()
    kx = k.reshape(2, 256, kvh, hd)
    for tok in range(254, 258):
        p, r = [1, 0][tok // 256], tok % 256
        pq, ps = kv_q68.kv_pack(kx[p, r].reshape(1, -1), kb)
        assert np.array_equal(cases.u16(kps[p, r].reshape(1, -1)), cases.u16(ps)) and _off_by_one_ok(kp[p, r].reshape(1, -1), pq, kb)
    tk.zero_(); tv.zero_()
    # (width 0 would return the temp untouched, cache.py get_kv_state; paged unpack converts [0, seqlen) whatever the width)
    ok, _ = cache.get_kv_state(0, 1, 0, 4, page_size=256, cache_seqlens=sl + 4, block_table=bt)
    torch.cuda.synchronize()
    okx = ok.view(2, 256, kvh, hd).cpu().numpy()
    for tok in (0, 255, 257):
        p, r = [1, 0][tok // 256], tok % 256
        want = kv_q68.kv_unpack(kp[p, r].reshape(1, -1), kps[p, r].reshape(1, -1), kb)
        assert np.array_equal(cases.u16(okx[p, r].reshape(1, -1)), cases.u16(want))
