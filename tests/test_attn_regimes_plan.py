"""tests/attn_regimes.py's restatement of the fused attention's launch arithmetic, pinned to the figures DESIGN.md §3.4
states, and the fp64 truth and query rotation the GPU tests build on (CPU only)."""
import numpy as np
import pytest

import attn_regimes as ar
import exl2_oracle as oracle
import kv_q68


@pytest.mark.parametrize("wbits,stage,stage_ring,sub", [(4, 512, 256, 128), (6, 320, 128, 64), (8, 256, 128, 64)])
@pytest.mark.parametrize("hd", [64, 128])
def test_stage_and_sub(wbits, hd, stage, stage_ring, sub):
    short = ar.plan(wbits, hd, 8, 1, 1, 4096, [100])
    long = ar.plan(wbits, hd, 8, 1, 1, 16384, [100])
    assert not short["ring"] and short["stage"] == stage and short["sub"] == sub
    assert long["ring"] and long["stage"] == stage_ring
    assert ar.plan(wbits, hd, 8, 1, 1, 8192, [100])["ring"] is False        # the ring starts above 8192 positions
    assert ar.plan(wbits, hd, 8, 1, 1, 8448, [100])["ring"] is True


def test_nsplit():
    assert ar.plan(4, 128, 32, 1, 1, 4096, [4095])["nsplit"] == 8
    for B in (9, 16):
        assert ar.plan(4, 128, 32, B, 1, 4096, [0] * B)["nsplit"] == 1
    assert ar.plan(4, 128, 32, 1, 2, 4096, [10])["nsplit"] == 1              # never with more than one query
    assert ar.plan(4, 128, 32, 1, 1, 1024, [10])["nsplit"] == 1              # nor over 1024 positions or fewer
    assert ar.plan(4, 128, 8, 1, 1, 16384, [10])["nsplit"] == 16             # capped at 16
    p = ar.plan(4, 128, 32, 1, 1, 4096, [4095])
    assert [(c["p_lo"], c["p_hi"]) for c in p["ctas"]] == [(z * 512, z * 512 + 512) for z in range(8)]
    p = ar.plan(4, 128, 8, 3, 1, 4096, [0, 511, 1500])                       # active chunks follow each sequence's length
    assert [c["ns_act"] for c in p["ctas"]] == [1, 1, 3, 3, 3]
    assert [(c["p_lo"], c["p_hi"]) for c in p["ctas"] if c["b"] == 2] == [(0, 501), (501, 1002), (1002, 1501)]


@pytest.mark.parametrize("wbits", [4, 6, 8])
def test_wide_head_layouts(wbits):
    """The 70B preset's 64 heads and a 28-head GQA-7 model (the regimes test_gpu_attn_regimes adds for them): 2 * 132 // 64 = 4
    chunks at B = 1, with the ring above 8192 positions; at B = 8 the 512 (head, sequence) CTAs outnumber the SMs and nothing
    splits; 264 // 28 = 9 chunks of 512 positions over a 4608-position cache."""
    p = ar.plan(wbits, 128, 64, 1, 1, 4096, [4095])
    assert p["nsplit"] == 4 and not p["ring"] and ar.branches(p, 1, 64, 1) >= {"merge", "global"}
    assert [(c["p_lo"], c["p_hi"]) for c in p["ctas"]] == [(z * 1024, z * 1024 + 1024) for z in range(4)]
    p = ar.plan(wbits, 128, 64, 1, 1, 16384, [16383])
    assert p["nsplit"] == 4 and p["ring"] and ar.branches(p, 1, 64, 1) >= {"merge", "ring"}
    p = ar.plan(wbits, 128, 64, 8, 1, 4096, [0, 1, 255, 256, 513, 1500, 3000, 4095])
    assert p["nsplit"] == 1 and ar.branches(p, 1, 64, 8) >= {"batched", "global"}
    p = ar.plan(wbits, 128, 28, 1, 1, 4608, [4607])
    assert p["nsplit"] == 9 and [(c["p_lo"], c["p_hi"]) for c in p["ctas"]] == [(z * 512, z * 512 + 512) for z in range(9)]
    assert 28 * 9 <= 2 * ar.H100_SMS and 64 * 4 <= 2 * ar.H100_SMS        # within the split-KV scratch bound (attn_q4.cu)


def _largest_fit(wbits, hd, q_len, B, H=32):
    pages = 1
    while ar.smem_bytes(wbits, hd, q_len, (pages + 1) * ar.PAGE, ar.nsplit_of(q_len, (pages + 1) * ar.PAGE, H, B))["fits"]:
        pages += 1
    return pages * ar.PAGE


@pytest.mark.parametrize("q_len,B", [(2, 1), (1, 9)])
def test_largest_cache_that_fits(q_len, B):
    """No split (q_len > 1, or H * B >= 2 * SMs): the score buffer holds the whole cache, so it bounds the context."""
    assert _largest_fit(4, 128, q_len, B) == 28928
    assert _largest_fit(8, 128, q_len, B) == 29696
    assert _largest_fit(6, 128, q_len, B) >= 28928


def test_no_format_needs_more_smem_than_q4():
    for ctx in (1024, 4096, 8192, 16384):
        for hd in (64, 128):
            q4 = ar.smem_bytes(4, hd, 2, ctx, 1)["smem"]
            assert ar.smem_bytes(6, hd, 2, ctx, 1)["smem"] <= q4 and ar.smem_bytes(8, hd, 2, ctx, 1)["smem"] <= q4


def test_cta_partition_covers_every_position_once():
    for wbits in (4, 6, 8):
        for hd in (64, 128):
            for q_len, ctx, seqlens in ((1, 16384, [0, 1, 511, 512, 9000, 16383]), (3, 12288, [0, 300, 12285]),
                                        (1, 4096, [0, 1, 255, 256, 4095])):
                p = ar.plan(wbits, hd, 8, len(seqlens), q_len, ctx, seqlens)
                for b, sl in enumerate(seqlens):
                    cs = [c for c in p["ctas"] if c["b"] == b]
                    cover = np.zeros(sl + q_len, dtype=int)
                    for c in cs:
                        cover[c["p_lo"]:c["p_hi"]] += 1
                        st = c["p_lo"] + c["n_st"]
                        assert c["c_hi"] - st == c["beyond"] >= 0
                        assert c["ntail"] * p["sub"] >= c["beyond"] > (c["ntail"] - 1) * p["sub"] or c["ntail"] == 0
                    assert (cover[:sl + 1] == 1).all()            # (with split, the chunks cover [0, seqlen]; q_len is 1)


def test_truth_and_rotation():
    rng = np.random.default_rng(0)
    B, q_len, H, KVH, hd, sl = 2, 3, 4, 2, 64, [5, 0]
    q = rng.normal(0, 1, (B, q_len, H, hd)).astype(np.float16)
    kn = rng.normal(0, 1, (B, q_len, KVH, hd)).astype(np.float16)
    vn = rng.normal(0, 1, (B, q_len, KVH, hd)).astype(np.float16)
    K = [rng.normal(0, 1, (s, KVH, hd)) for s in sl]
    V = [rng.normal(0, 1, (s, KVH, hd)) for s in sl]
    got = ar.attention_truth(q, kn, vn, K, V, sl, 0.125)
    for b in range(B):
        for i in range(q_len):
            for h in range(H):
                kk = np.concatenate([K[b][:, h // 2], kn[b, :i + 1, h // 2]]).astype(np.float64)
                vv = np.concatenate([V[b][:, h // 2], vn[b, :i + 1, h // 2]]).astype(np.float64)
                s = kk @ q[b, i, h].astype(np.float64) * 0.125
                p = np.exp(s - s.max())
                assert np.allclose(got[b, i, h], (p / p.sum()) @ vv, rtol=1e-12, atol=1e-14)
    # the fp32 rotation is the stored-domain Hadamard: q . x = (H q) . y / 32 for x = H y / 32
    x = rng.normal(0, 1, hd).astype(np.float16)
    rq = ar.rotate_q_fp32(x, np.float32(32.0)).astype(np.float64)
    Hm = np.array([[(-1) ** bin(i & j).count("1") for j in range(32)] for i in range(32)], dtype=np.float64)
    y = np.stack([Hm @ x.astype(np.float64)[0::2], Hm @ x.astype(np.float64)[1::2]], -1).reshape(hd)   # the oracle's butterfly, in fp64
    assert np.allclose(rq, y, rtol=1e-6, atol=1e-5)
    assert np.allclose(oracle._hadamard32_interleaved(x.reshape(1, 64)).astype(np.float64).reshape(hd), y, rtol=4e-3, atol=1e-2)
    # a stored one-hot dequantises to +-A/32 on one Hadamard row
    for bits in (4, 8):
        d = ar.key_direction(hd, bits, 37)
        assert np.count_nonzero(d) == 32 and np.allclose(np.abs(d[d != 0]), ar.one_hot_amp(bits) / 32)
        row = ar.s_one_hot_row(hd, bits, 37, neg=True)
        dn = kv_q68.kv_unpack(row[None], np.ones((1, hd // 32), np.float16), bits)[0].astype(np.float64)
        assert np.allclose(dn * ar.one_hot_amp(bits), -d * 8)
