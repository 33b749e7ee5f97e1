"""GPU parity tests: RMSNorm, RoPE, silu*mul, Q4 K/V cache and the fused attention / MLP blocks vs the oracle."""
import numpy as np
import pytest
import torch

import cases
import exl2_oracle as oracle
import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _ulp_diff(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """distance in fp16 representable steps (sign-magnitude -> monotone integer)."""
    def key(x):
        u = np.ascontiguousarray(x, dtype=np.float16).view(np.uint16).astype(np.int32)
        return np.where(u & 0x8000, -(u & 0x7FFF), u & 0x7FFF)
    return np.abs(key(a) - key(b))


@pytest.mark.parametrize("rows,dim", [(1, 4096), (3, 2048), (17, 5632), (2, 8192), (5, 64)])
def test_rms_norm(rows, dim):
    from exllamav2_b200 import ext as ext_c
    rng = np.random.default_rng(rows * 31 + dim)
    x = rng.normal(0, 1.5, size=(rows, dim)).astype(np.float16)
    w = (1 + 0.1 * rng.normal(size=(dim,))).astype(np.float16)
    xt, wt = torch.from_numpy(x).to(DEV), torch.from_numpy(w).to(DEV)
    y = torch.empty_like(xt)
    ext_c.rms_norm(xt, wt, y, 1e-5)
    want = oracle.rms_norm(x, w, 1e-5)
    d = _ulp_diff(y.cpu().numpy(), want)
    assert d.max() <= 1, f"max ulp diff {d.max()}"           # tolerance: 1 fp16 ulp (fp32 summation order)
    assert (d > 0).mean() < 0.01
    ext_c.rms_norm_(xt, wt, 1e-5)                             # in-place form
    assert torch.equal(xt, y)


def test_rms_norm_inf_clamp():
    from exllamav2_b200 import ext as ext_c
    x = np.zeros((1, 64), dtype=np.float16)
    x[0, 3] = np.inf
    x[0, 5] = 2.0
    w = np.ones((64,), dtype=np.float16)
    xt = torch.from_numpy(x).to(DEV)
    y = torch.empty_like(xt)
    ext_c.rms_norm(xt, torch.from_numpy(w).to(DEV), y, 1e-5)
    assert np.array_equal(cases.u16(y.cpu().numpy()), cases.u16(oracle.rms_norm(x, w, 1e-5)))


@pytest.mark.parametrize("neox", [True, False])
@pytest.mark.parametrize("batch,q_len,heads,hd", [(1, 1, 32, 128), (2, 5, 4, 64), (1, 7, 8, 128)])
def test_rope(neox, batch, q_len, heads, hd):
    """Bit-exact: same fp16 op order as cuda/rope.cu:52-67 / :111-122."""
    from exllamav2_b200 import ext as ext_c
    rng = np.random.default_rng(batch * 100 + q_len * 10 + heads)
    sin, cos = oracle.rope_tables(hd, 256)
    x = rng.normal(0, 1, size=(batch, q_len, heads * hd)).astype(np.float16)
    past_len = 13
    offsets = np.array([0, 3][:batch], dtype=np.int32)
    xt = torch.from_numpy(x).to(DEV)
    ext_c.rope_(xt, torch.from_numpy(sin).to(DEV), torch.from_numpy(cos).to(DEV), past_len, heads, hd,
                torch.from_numpy(offsets).to(DEV), neox)
    fn = oracle.rope_neox if neox else oracle.rope_gptj
    want = np.stack([fn(x[b].reshape(q_len, heads, hd), sin, cos, past_len + offsets[b] + np.arange(q_len)).reshape(q_len, heads * hd)
                     for b in range(batch)])
    assert np.array_equal(cases.u16(xt.cpu().numpy()), cases.u16(want))
    # past_len == -1: position comes from past_lens alone (rope.cu:39-43); no offsets tensor -> past_len only
    from exllamav2_b200.ext import none_tensor
    xt2 = torch.from_numpy(x).to(DEV)
    ext_c.rope_(xt2, torch.from_numpy(sin).to(DEV), torch.from_numpy(cos).to(DEV), past_len, heads, hd, none_tensor, neox)
    want2 = np.stack([fn(x[b].reshape(q_len, heads, hd), sin, cos, past_len + np.arange(q_len)).reshape(q_len, heads * hd)
                      for b in range(batch)])
    assert np.array_equal(cases.u16(xt2.cpu().numpy()), cases.u16(want2))


@pytest.mark.parametrize("neox", [True, False])
@pytest.mark.parametrize("hd", [64, 128])
def test_rope_partial_rotary(neox, hd):
    """sincos_size = head_dim / 2 (partial rotary): the first sincos_size dimensions of every head rotate, the rest pass
    through untouched; bit-exact against the oracle with its rotary width, per-sequence offsets and past_len = -1."""
    from exllamav2_b200 import ext as ext_c
    batch, q_len, heads, rot = 3, 4, 4, hd // 2
    rng = np.random.default_rng(hd + neox)
    sin, cos = oracle.rope_tables(rot, 64)
    x = rng.normal(0, 1, size=(batch, q_len, heads * hd)).astype(np.float16)
    fn = oracle.rope_neox if neox else oracle.rope_gptj
    st, ct = torch.from_numpy(sin).to(DEV), torch.from_numpy(cos).to(DEV)
    for past_len, offs in ((5, np.array([0, 7, 2], dtype=np.int32)), (-1, np.array([11, 0, 3], dtype=np.int32))):
        xt = torch.from_numpy(x).to(DEV)
        ext_c.rope_(xt, st, ct, past_len, heads, hd, torch.from_numpy(offs).to(DEV), neox)
        base = offs if past_len == -1 else past_len + offs
        want = np.stack([fn(x[b].reshape(q_len, heads, hd), sin, cos, base[b] + np.arange(q_len), rot).reshape(q_len, heads * hd)
                         for b in range(batch)])
        got = xt.cpu().numpy()
        assert np.array_equal(cases.u16(got), cases.u16(want)), f"past_len {past_len}"
        assert np.array_equal(cases.u16(got.reshape(batch, q_len, heads, hd)[..., rot:]),
                              cases.u16(x.reshape(batch, q_len, heads, hd)[..., rot:]))


def test_act_mul():
    from exllamav2_b200 import ext as ext_c
    rng = np.random.default_rng(3)
    g = rng.normal(0, 2, size=(5, 11008)).astype(np.float16)
    u = rng.normal(0, 1, size=(5, 11008)).astype(np.float16)
    gt = torch.from_numpy(g).to(DEV)
    ext_c.act_mul(gt, torch.from_numpy(u).to(DEV))
    want = oracle.silu_mul(g, u).astype(np.float32)
    got = gt.float().cpu().numpy()
    # hexp / hrcp are approximate intrinsics (q_mlp_activation.cuh:13-22): a few fp16 ulp
    assert np.allclose(got, want, rtol=4e-3, atol=2e-3)


def test_act_mul_gelu():
    """act_gelu: tanh-form GELU in fp32 (tanh.approx on the GPU), rounded to fp16, times up in fp16 -- a few fp16 ulp from the
    exact-tanh oracle.  The gate spans the tanh saturation on both sides and the cubic term's range."""
    from exllamav2_b200 import ext as ext_c
    rng = np.random.default_rng(4)
    g = rng.normal(0, 2, size=(5, 11008)).astype(np.float16)
    g[0, :64] = np.linspace(-12, 12, 64).astype(np.float16)
    u = rng.normal(0, 1, size=(5, 11008)).astype(np.float16)
    gt = torch.from_numpy(g).to(DEV)
    ext_c.act_mul(gt, torch.from_numpy(u).to(DEV), act_gelu=True)
    want = oracle.gelu_mul(g, u)
    got = gt.cpu().numpy()
    # (tanh.approx has ~2^-11 relative error; where tanh(t) -> -1 the 1 + tanh cancellation turns that into an absolute error)
    assert np.allclose(got.astype(np.float32), want.astype(np.float32), rtol=4e-3, atol=2e-3)
    # not silu: the two activations differ by far more than the tolerance on this range
    assert not np.allclose(got.astype(np.float32), oracle.silu_mul(g, u).astype(np.float32), rtol=4e-3, atol=2e-3)


@pytest.mark.parametrize("shape", [(2, 16, 32, 128), (1, 8, 4, 64), (3, 4, 8, 128)])
def test_kv_q4_roundtrip_nonpaged(shape):
    """pack -> (compare with oracle) -> unpack -> (compare with oracle); [batch, seq, heads, head_dim]."""
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200.ext import none_tensor
    B, S, H, D = shape
    rng = np.random.default_rng(sum(shape))
    k = rng.normal(0, 1, size=shape).astype(np.float16)
    v = rng.normal(0, 2, size=shape).astype(np.float16)
    kt, vt = torch.from_numpy(k).to(DEV), torch.from_numpy(v).to(DEV)
    kq = torch.zeros((B, S, H, D // 2), dtype=torch.uint8, device=DEV)
    vq = torch.zeros_like(kq)
    ks = torch.zeros((B, S, H, D // 32), dtype=torch.half, device=DEV)
    vs = torch.zeros_like(ks)
    ext_c.fp16_to_q_kv(kt, kq, ks, vt, vq, vs, B, 0, S, 0, none_tensor, none_tensor, 4)
    for src, q, s in ((k, kq, ks), (v, vq, vs)):
        pq, ps = oracle.kv_pack_q4(src.reshape(B, S * H * D))
        got_q = q.cpu().numpy().reshape(B, -1)
        got_s = s.cpu().numpy().reshape(B, -1)
        assert np.array_equal(cases.u16(got_s), cases.u16(ps)), "scales differ"
        lo = (got_q & 15).astype(int) - (pq & 15).astype(int)
        hi = (got_q >> 4).astype(int) - (pq >> 4).astype(int)
        # __h2div is rcp-based: a handful of values may land on the other side of a rounding tie
        assert np.abs(lo).max() <= 1 and np.abs(hi).max() <= 1
        assert (np.count_nonzero(lo) + np.count_nonzero(hi)) <= 1e-3 * src.size
    ko, vo = torch.zeros_like(kt), torch.zeros_like(vt)
    ext_c.q_to_fp16_kv(kq, ko, ks, vq, vo, vs, B, 0, S, 0, none_tensor, none_tensor, 4)
    for q, s, o in ((kq, ks, ko), (vq, vs, vo)):
        want = oracle.kv_unpack_q4(q.cpu().numpy().reshape(B, -1), s.cpu().numpy().reshape(B, -1)).reshape(shape)
        assert np.array_equal(cases.u16(o.cpu().numpy()), cases.u16(want)), "unpack is not bit-exact"
    # quantisation error sanity (Q4 with Hadamard: ~7% rms of the signal)
    err = (ko.float() - kt.float()).norm() / kt.float().norm()
    assert err < 0.15


def test_kv_q4_partial_range_leaves_rest_untouched():
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200.ext import none_tensor
    B, S, H, D = 2, 12, 32, 128
    k = torch.randn((B, S, H, D), dtype=torch.half, device=DEV)
    kq = torch.full((B, S, H, D // 2), 0xAB, dtype=torch.uint8, device=DEV)
    ks = torch.full((B, S, H, D // 32), 7.0, dtype=torch.half, device=DEV)
    ext_c.fp16_to_q_kv(k, kq, ks, none_tensor, none_tensor, none_tensor, B, 5, 3, 0, none_tensor, none_tensor, 4)
    assert (kq[:, :5] == 0xAB).all() and (kq[:, 8:] == 0xAB).all() and (ks[:, :5] == 7.0).all() and (ks[:, 8:] == 7.0).all()
    assert not (kq[:, 5:8] == 0xAB).all()


def test_kv_q4_paged():
    """Paged form (cache.cu:143-223 / :324-401): block_table maps (seq, page) -> physical page of 256 tokens."""
    from exllamav2_b200 import ext as ext_c
    page, H, D = 256, 4, 64                       # TinyLlama-like: dim 256 (not a multiple of 512)
    pages_total = 6
    rng = np.random.default_rng(9)
    block_table = np.array([[4, 1], [0, 5]], dtype=np.int32)
    seqlens = np.array([250, 3], dtype=np.int32)  # seq 0 crosses into its second page with q_len 10
    q_len = 10
    k = rng.normal(0, 1, size=(pages_total, page, H, D)).astype(np.float16)
    v = rng.normal(0, 1, size=(pages_total, page, H, D)).astype(np.float16)
    kt, vt = torch.from_numpy(k).to(DEV), torch.from_numpy(v).to(DEV)
    kq = torch.zeros((pages_total, page, H, D // 2), dtype=torch.uint8, device=DEV)
    vq = torch.zeros_like(kq)
    ks = torch.zeros((pages_total, page, H, D // 32), dtype=torch.half, device=DEV)
    vs = torch.zeros_like(ks)
    bt, sl = torch.from_numpy(block_table).to(DEV), torch.from_numpy(seqlens).to(DEV)
    ext_c.fp16_to_q_kv(kt, kq, ks, vt, vq, vs, 2, 0, q_len, page, sl, bt, 4)
    dim = H * D
    touched = torch.zeros((pages_total, page), dtype=torch.bool)
    for s in range(2):
        a, b = int(seqlens[s]), int(seqlens[s]) + q_len
        while (a * dim) % 512: a -= 1
        while (b * dim) % 512: b += 1
        for tok in range(a, b):
            p = block_table[s, tok // page]
            touched[p, tok % page] = True
            pq, ps = oracle.kv_pack_q4(k[p, tok % page].reshape(1, -1))
            assert np.array_equal(cases.u16(ks[p, tok % page].cpu().numpy().reshape(1, -1)), cases.u16(ps))
    assert (ks.cpu()[~touched] == 0).all(), "pack wrote outside the token range"
    # unpack everything up to seqlen + q_len
    sl2 = torch.from_numpy(seqlens + q_len).to(DEV)
    ko, vo = torch.zeros_like(kt), torch.zeros_like(vt)
    ext_c.q_to_fp16_kv(kq, ko, ks, vq, vo, vs, 2, 0, 0, page, sl2, bt, 4)
    for s in range(2):
        for tok in (int(seqlens[s]), int(seqlens[s]) + q_len - 1):
            p = block_table[s, tok // page]
            want = oracle.kv_unpack_q4(kq[p, tok % page].cpu().numpy().reshape(1, -1), ks[p, tok % page].cpu().numpy().reshape(1, -1))
            assert np.array_equal(cases.u16(ko[p, tok % page].cpu().numpy().reshape(1, -1)), cases.u16(want))



@pytest.mark.parametrize("H,KVH,hd,q_len,seqlens", [
    (8, 8, 128, 1, [300, 0]),          # crosses a page; an empty sequence
    (8, 2, 64, 3, [17, 255]),          # GQA, several new rows, append runs over a page end
    (4, 4, 128, 8, [511, 5]),
])
def test_paged_attn_decode_q4(H, KVH, hd, q_len, seqlens):
    """Fused Q4 attention == oracle: pack the new rows (fp16_to_q_kv arithmetic, bit-exact cache contents), then
    softmax(q K^T / sqrt(hd)) V in fp64 over the oracle-dequantised cached rows plus the new rows in fp16 -- the step
    that appends a row attends it unquantised, as flash_attn_with_kvcache does in the reference (attn.py:602-621).
    Tolerance 2e-3 relative L2 (the reference pipeline rounds the dequantised K/V to fp16; this kernel keeps fp32)."""
    from exllamav2_b200 import ext as ext_c
    page, pps = 256, 3
    B = len(seqlens)
    rng = np.random.default_rng(31)
    pages_total = B * pps + 1
    block_table = rng.permutation(pages_total)[:B * pps].reshape(B, pps).astype(np.int32)
    past_k = rng.normal(0, 1, size=(pages_total, page, KVH, hd)).astype(np.float16)
    past_v = rng.normal(0, 1, size=(pages_total, page, KVH, hd)).astype(np.float16)
    kq0, ks0 = oracle.kv_pack_q4(past_k)
    vq0, vs0 = oracle.kv_pack_q4(past_v)
    q = rng.normal(0, 1, size=(B, q_len, H, hd)).astype(np.float16)
    kn = rng.normal(0, 1, size=(B, q_len, KVH, hd)).astype(np.float16)
    vn = rng.normal(0, 1, size=(B, q_len, KVH, hd)).astype(np.float16)
    t = lambda a: torch.from_numpy(a).to(DEV)
    kq, ks, vq, vs = t(kq0.copy()), t(ks0.copy()), t(vq0.copy()), t(vs0.copy())
    out = torch.zeros((B, q_len, H, hd), dtype=torch.half, device=DEV)
    sl = t(np.array(seqlens, dtype=np.int32))
    ext_c.paged_attn_decode_q4(t(q), t(kn), t(vn), kq, ks, vq, vs, sl, t(block_table), out, 1.0 / np.sqrt(hd))
    torch.cuda.synchronize()
    kq1, ks1, vq1, vs1 = kq.cpu().numpy(), ks.cpu().numpy(), vq.cpu().numpy(), vs.cpu().numpy()
    got = out.cpu().numpy()
    # 1. the appended rows are exactly what fp16_to_q_kv stores; nothing else moved
    want_kq, want_ks, want_vq, want_vs = kq0.copy(), ks0.copy(), vq0.copy(), vs0.copy()
    nkq, nks = oracle.kv_pack_q4(kn)
    nvq, nvs = oracle.kv_pack_q4(vn)
    for b in range(B):
        for i in range(q_len):
            pos = seqlens[b] + i
            pg = block_table[b, pos // page]
            want_kq[pg, pos % page], want_ks[pg, pos % page] = nkq[b, i], nks[b, i]
            want_vq[pg, pos % page], want_vs[pg, pos % page] = nvq[b, i], nvs[b, i]
    assert np.array_equal(kq1, want_kq) and np.array_equal(vq1, want_vq)
    assert np.array_equal(cases.u16(ks1), cases.u16(want_ks)) and np.array_equal(cases.u16(vs1), cases.u16(want_vs))
    # 2. attention over the dequantised cache
    kd = oracle.kv_unpack_q4(kq1, ks1).astype(np.float64)
    vd = oracle.kv_unpack_q4(vq1, vs1).astype(np.float64)
    group = H // KVH
    for b in range(B):
        for i in range(q_len):
            n = seqlens[b] + i + 1
            rows = [(block_table[b, p // page], p % page) for p in range(seqlens[b])]
            for h in range(H):
                K = np.stack([kd[pg, r, h // group] for pg, r in rows] + [kn[b, j, h // group].astype(np.float64) for j in range(i + 1)])
                V = np.stack([vd[pg, r, h // group] for pg, r in rows] + [vn[b, j, h // group].astype(np.float64) for j in range(i + 1)])
                s = K @ q[b, i, h].astype(np.float64) / np.sqrt(hd)
                pr = np.exp(s - s.max())
                ref = (pr / pr.sum()) @ V
                err = oracle.rel_l2(got[b, i, h].astype(np.float64), ref)
                assert err < 2e-3, (b, i, h, err)


# ---- fused blocks ---------------------------------------------------------------------------------------------------

def _lin(w_np, K, N):
    from exllamav2_b200.linear import ExLlamaV2Linear, load_tensor_dict
    lin = ExLlamaV2Linear(K, N, has_bias="bias" in w_np, device=DEV)
    lin.load(load_tensor_dict(w_np, DEV))
    return lin


@pytest.mark.parametrize("rows", [1, 3, 8, 9, 11])
@pytest.mark.parametrize("gptq", [False, True])
def test_q_attn_block(rows, gptq):
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200.ext import none_tensor
    hidden, heads, kv_heads, hd = 512, 8, 2, 64
    mk = (lambda K, N, seed: synth.make_gptq(K, N, 128, seed=seed, act_order=True)) if gptq else \
         (lambda K, N, seed: synth.make_exl2(K, N, (5, 4), (0.1, 0.9), 64, seed=seed))
    recon = oracle.gptq_reconstruct if gptq else oracle.exl2_reconstruct
    wq, wk, wv, wo = mk(hidden, heads * hd, 1), mk(hidden, kv_heads * hd, 2), mk(hidden, kv_heads * hd, 3), mk(heads * hd, hidden, 4)
    Wq, Wk, Wv, Wo = recon(wq), recon(wk), recon(wv), recon(wo)
    lq, lk, lv, lo = _lin(wq, hidden, heads * hd), _lin(wk, hidden, kv_heads * hd), _lin(wv, hidden, kv_heads * hd), _lin(wo, heads * hd, hidden)
    rng = np.random.default_rng(rows)
    norm_w = (1 + 0.1 * rng.normal(size=(hidden,))).astype(np.float16)
    sin, cos = oracle.rope_tables(hd, 128)
    x = rng.normal(0, 1, size=(1, rows, hidden)).astype(np.float16)
    nw = torch.from_numpy(norm_w).to(DEV)
    h = ext_c.make_q_attn(nw, none_tensor, True, False, 1e-5, lq.q_handle, lk.q_handle, lv.q_handle, lo.q_handle,
                          none_tensor, none_tensor, 64, hidden, heads, kv_heads, hd, 128, True, 2, hd,
                          none_tensor, none_tensor, none_tensor, none_tensor, False, True)
    xt = torch.from_numpy(x).to(DEV)
    q = torch.empty((1, rows, heads * hd), dtype=torch.half, device=DEV)
    k = torch.empty((1, rows, kv_heads * hd), dtype=torch.half, device=DEV)
    v = torch.empty_like(k)
    past = 7
    ext_c.q_attn_forward_1(h, xt, 1, rows, past, none_tensor, q, k, v, torch.from_numpy(sin).to(DEV), torch.from_numpy(cos).to(DEV))
    xn = oracle.rms_norm(x[0], norm_w, 1e-5)
    pos = past + np.arange(rows)
    q_t = oracle.gemm_truth(xn, Wq).astype(np.float16)
    k_t = oracle.gemm_truth(xn, Wk).astype(np.float16)
    v_t = oracle.gemm_truth(xn, Wv).astype(np.float16)
    q_w = oracle.rope_neox(q_t.reshape(rows, heads, hd), sin, cos, pos).reshape(rows, -1)
    k_w = oracle.rope_neox(k_t.reshape(rows, kv_heads, hd), sin, cos, pos).reshape(rows, -1)
    for got, want, nm in ((q, q_w, "q"), (k, k_w, "k"), (v, v_t, "v")):
        err = oracle.rel_l2(got[0].cpu().numpy(), want)
        assert err <= 1.5e-3, f"{nm}: rel_l2 {err:.2e}"       # one extra fp16 rounding (norm) + rope roundings
    # part 2: x += attn_out @ Wo
    attn_out = rng.normal(0, 1, size=(1, rows, heads * hd)).astype(np.float16)
    x2 = xt.clone()
    ext_c.q_attn_forward_2(h, x2, torch.from_numpy(attn_out).to(DEV), 1, rows)
    want = oracle.gemm_truth(attn_out[0], Wo, None, x[0])
    assert oracle.rel_l2(x2[0].cpu().numpy(), want) <= 5e-4
    ext_c.free_q_attn(h)
    for l in (lq, lk, lv, lo): l.unload()


def _q_mlp_block(rows, act_gelu, bias, share_perm=False):
    """rows 1: integer GEMV with act*mul as the down launch's prologue when gate and up share their row permutation (as converted
    checkpoints do), otherwise the one-row wgmma pass; 2..8: one wgmma pass with the paired gate|up
    epilogue; 9..16: two passes (9: an 8-row pass and a one-row tail pass); > 16: dense GEMMs + act_mul."""
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200.ext import none_tensor
    hidden, inter = 256, 704       # 704 = 11 strips of 64
    wg = synth.make_exl2(hidden, inter, (4, 3), (0.1, 0.9), 128, seed=5, scale_max_range=(0.02, 0.08), bias=bias)
    wu = synth.make_exl2(hidden, inter, (4,), (1.0,), 32, seed=6, scale_max_range=(0.02, 0.08), bias=bias)
    wd = synth.make_exl2(inter, hidden, (6, 5), (0.1, 0.9), 32, seed=7, scale_max_range=(0.02, 0.08))
    if share_perm:
        wu["q_invperm"] = wg["q_invperm"].copy()
    Wg, Wu, Wd = oracle.exl2_reconstruct(wg), oracle.exl2_reconstruct(wu), oracle.exl2_reconstruct(wd)
    lg, lu, ld = _lin(wg, hidden, inter), _lin(wu, hidden, inter), _lin(wd, inter, hidden)
    rng = np.random.default_rng(rows + 50)
    norm_w = (1 + 0.1 * rng.normal(size=(hidden,))).astype(np.float16)
    x = rng.normal(0, 1, size=(rows, hidden)).astype(np.float16)
    ta = torch.empty((rows, inter), dtype=torch.half, device=DEV)
    tb = torch.empty_like(ta)
    nw = torch.from_numpy(norm_w).to(DEV)          # must outlive the handle (raw pointer, like the reference)
    h = ext_c.make_q_mlp(nw, none_tensor, True, 1e-5, lg.q_handle, lu.q_handle, ld.q_handle,
                         none_tensor, ta, tb, none_tensor, 64, act_gelu, True, none_tensor, none_tensor, False, True)
    xt = torch.from_numpy(x).to(DEV)
    ext_c.q_mlp_forward_(h, xt)
    xn = oracle.rms_norm(x, norm_w, 1e-5)
    g = oracle.gemm_truth(xn, Wg, wg.get("bias")).astype(np.float16)
    u = oracle.gemm_truth(xn, Wu, wu.get("bias")).astype(np.float16)
    a = (oracle.gelu_mul if act_gelu else oracle.silu_mul)(g, u)
    # intermediate act(gate)*up (approximate hexp/hrcp, tanh.approx); the single-row path never materialises it
    if rows > 1:
        assert oracle.rel_l2(ta.cpu().numpy(), a) <= 3e-3
        other = (oracle.silu_mul if act_gelu else oracle.gelu_mul)(g, u)
        assert oracle.rel_l2(ta.cpu().numpy(), other) > 1e-2, "the other activation fits as well: the test cannot tell them apart"
    want = oracle.gemm_truth(a, Wd, None, x)
    assert oracle.rel_l2(xt.cpu().numpy(), want) <= 3e-3
    ext_c.free_q_mlp(h)
    for l in (lg, lu, ld): l.unload()


@pytest.mark.parametrize("rows", [1, 2, 8, 9, 13, 40])
def test_q_mlp_block(rows):
    _q_mlp_block(rows, False, False)


@pytest.mark.parametrize("rows", [1, 2, 8, 9, 13, 40])
@pytest.mark.parametrize("share_perm", [False, True], ids=["own_perm", "shared_perm"])
def test_q_mlp_block_gelu(rows, share_perm):
    _q_mlp_block(rows, True, False, share_perm)


@pytest.mark.parametrize("act_gelu", [False, True])
@pytest.mark.parametrize("rows", [1, 5, 12, 40])
def test_q_mlp_block_bias(rows, act_gelu):
    """gate / up linears with a bias: added in fp32 before the fp16 rounding that feeds the activation"""
    _q_mlp_block(rows, act_gelu, True, share_perm=True)
