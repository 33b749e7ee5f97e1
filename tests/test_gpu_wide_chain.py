"""Chained launches of 9..64 rows (csrc/gemm_tc.cu's 32- and 64-row wgmma tiles) against fp64, entry point by entry point.

A chained launch runs all its rows in one pass on the narrowest token tile that holds them (tests/wide_plan.py tile_for):
9..32 rows on wgmma.m64n32k16, 33..64 on m64n64k16, each producer scattering into its consumers' 64-row activation buffers.
Covered here, on every format the wgmma kernel can stage and at rows 9, 16, 17, 31, 32, 33, 40, 63, 64:
  * every chained entry point (q_attn_forward_2_ex -> q_mlp_forward_ex -> q_attn_forward_1_ex with RoPE at ragged per-sequence
    positions, and q_mlp_forward_ex -> gemm_half_q_half_prepared) against an fp64 composition from the kernel's previous fp16
    output (<= 1.5e-3 rel-L2, <= 4e-3 on any row) and against the plain forms (<= 2e-3), as test_gpu_tc_paths does at 2..8;
  * bias, residual, SiLU and GELU products;
  * fused RoPE, GPT-J and NeoX, head dims 64 and 128, full and partial width, past_len fixed or -1 with ragged per-sequence
    lengths: BIT-EXACT against oracle rotation of the same launch's un-rotated output (a rope_style = 0 handle on the same
    matrices runs the identical launch on the same activation buffer);
  * the refusals: 65 rows on every chained entry point, and groups above 128 rows at 9..64, neither touching x;
  * state: an 8-row chained graph captured before a wide launch replays to eager's bits after it, a captured wide step equals
    eager, and two streams get distinct wide scratch.
"""
import math

import numpy as np
import pytest
import torch

import exl2_oracle as oracle
import test_gpu_group_structures as gs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROWS = [9, 16, 17, 31, 32, 33, 40, 63, 64]
STAGEABLE = {f: gs.FORMATS[f][0] for f, v in gs.FORMATS.items() if v[3]}
STAGEABLE.update({"exl2_54_g128": ((5, 4), (0.1, 0.9), 128), "gptq_g128_act": ("gptq", 128, True)})


def _lin(K, N, plan, seed, perm_seed=None, bias=False):
    from exllamav2_b200 import synthetic
    from exllamav2_b200.linear import ExLlamaV2Linear
    w = synthetic.random_linear(K, N, plan, device=DEV, seed=seed, weight_std=1.0 / math.sqrt(K), perm_seed=perm_seed)
    if bias:
        g = torch.Generator(device=DEV).manual_seed(seed)
        w["bias"] = (0.1 * torch.randn(N, device=DEV, generator=g)).half()
    lin = ExLlamaV2Linear(K, N, has_bias=bias, device=DEV)
    lin.load(w)
    lin.test_bias = w.get("bias")
    return lin


def _rel(got, want):
    return (torch.linalg.norm(got.double() - want) / torch.linalg.norm(want)).item()


def _row_rel(got, want):
    d = got.double() - want
    return (torch.linalg.norm(d, dim=-1) / torch.linalg.norm(want, dim=-1).clamp_min(1e-30)).max().item()


def _t_norm(x, w, eps=1e-5):
    xf = x.double()
    return xf * w.double() / torch.sqrt((xf * xf).mean(-1, keepdim=True) + eps)


def _batch(rows):
    """(batch, q_len): one new token per sequence, except 40 rows as 5 sequences x 8 tokens"""
    return (5, 8) if rows == 40 else (rows, 1)


class Block:
    """One attention + MLP block and a head on a format, with the chains of the decoder step."""

    def __init__(self, fmt, hidden=512, inter=1408, heads=8, kv_heads=4, hd=64, gelu=False, bias=False, rope_style=2, rot=None):
        from exllamav2_b200 import ext as ext_c
        from exllamav2_b200.ext import none_tensor
        plan = STAGEABLE.get(fmt, gs.FORMATS.get(fmt, (None,))[0])
        if fmt == "exl2_4b_g128_k1376":
            inter = 1376                     # down's K ends in a short group of 96 rows
        self.hidden, self.inter, self.heads, self.kv_heads, self.hd = hidden, inter, heads, kv_heads, hd
        self.rot = rot or hd
        mk = lambda K, N, s, p=None, b=False: _lin(K, N, plan, s, p, b)
        self.lq, self.lk, self.lv = mk(hidden, heads * hd, 51, 51), mk(hidden, kv_heads * hd, 52, 51), mk(hidden, kv_heads * hd, 53, 51)
        self.lo = mk(heads * hd, hidden, 54, None, bias)
        self.lg, self.lu, self.ld = mk(hidden, inter, 55, 55, bias), mk(hidden, inter, 56, 55, bias), mk(inter, hidden, 57)
        self.lh = mk(hidden, 1024, 58)
        self.lins = [self.lq, self.lk, self.lv, self.lo, self.lg, self.lu, self.ld, self.lh]
        rng = np.random.default_rng(7)
        self.n1, self.n2, self.n3 = (torch.from_numpy((1 + 0.1 * rng.normal(size=(hidden,))).astype(np.float16)).to(DEV) for _ in range(3))
        self.ta = torch.empty((64 * 8, inter), dtype=torch.half, device=DEV)
        self.tb = torch.empty_like(self.ta)
        self.hat = {}
        for style in {0, rope_style}:
            self.hat[style] = ext_c.make_q_attn(self.n1, none_tensor, True, False, 1e-5, self.lq.q_handle, self.lk.q_handle,
                                                self.lv.q_handle, self.lo.q_handle, none_tensor, none_tensor, 64, hidden, heads,
                                                kv_heads, hd, 512, True, style, self.rot, none_tensor, none_tensor, none_tensor,
                                                none_tensor, False, True)
        self.style = rope_style
        self.hml = ext_c.make_q_mlp(self.n2, none_tensor, True, 1e-5, self.lg.q_handle, self.lu.q_handle, self.ld.q_handle,
                                    none_tensor, self.ta, self.tb, none_tensor, 64, gelu, True, none_tensor, none_tensor, False, True)
        self.gelu = gelu
        self.chain_mlp = ext_c.make_chain([self.lg.q_handle, self.lu.q_handle], self.n2)
        self.chain_attn = ext_c.make_chain([self.lq.q_handle, self.lk.q_handle, self.lv.q_handle], self.n1)
        self.chain_head = ext_c.make_chain([self.lh.q_handle], self.n3)
        self.W = {n: l.get_weight_tensor_dq().double() for n, l in zip("qkvoguda", self.lins)}
        self.B = {n: (l.test_bias.double() if l.test_bias is not None else 0.0) for n, l in zip("qkvoguda", self.lins)}

    def close(self):
        from exllamav2_b200 import ext as ext_c
        for h in self.hat.values():
            ext_c.free_q_attn(h)
        ext_c.free_q_mlp(self.hml)
        for l in self.lins:
            l.unload()


def _mlp_truth(b, x):
    xn = _t_norm(x, b.n2)
    g, u = (xn @ b.W["g"] + b.B["g"]).half().cpu().numpy(), (xn @ b.W["u"] + b.B["u"]).half().cpu().numpy()
    act = oracle.gelu_mul(g, u) if b.gelu else oracle.silu_mul(g, u)
    return x.double() + torch.from_numpy(act).to(DEV).double() @ b.W["d"]


def _chained_step(b, rows, past_lens, sin, cos, x0, ao):
    """o_proj -> MLP -> q|k|v (RoPE) chained, then o_proj -> MLP -> head; returns the stage outputs"""
    from exllamav2_b200 import ext as ext_c
    batch, q_len = _batch(rows)
    new = lambda n: torch.empty((batch, q_len, n), dtype=torch.half, device=DEV)
    xb = x0.clone()
    ext_c.q_attn_forward_2_ex(b.hat[b.style], xb, ao, batch, q_len, False, b.chain_mlp)
    xb1 = xb.clone().view(rows, -1)
    ext_c.q_mlp_forward_ex(b.hml, xb.view(rows, -1), True, b.chain_attn)
    q, k, v = new(b.heads * b.hd), new(b.kv_heads * b.hd), new(b.kv_heads * b.hd)
    ext_c.q_attn_forward_1_ex(b.hat[b.style], None, batch, q_len, -1, past_lens, q, k, v, sin, cos, True)
    xc = x0.clone()
    ext_c.q_attn_forward_2_ex(b.hat[b.style], xc, ao, batch, q_len, False, b.chain_mlp)
    ext_c.q_mlp_forward_ex(b.hml, xc.view(rows, -1), True, b.chain_head)
    lg = torch.empty((rows, 1024), dtype=torch.half, device=DEV)
    ext_c.gemm_half_q_half_prepared(b.lh.q_handle, lg, True, 1e-5)
    return dict(x1=xb1, x2=xb.view(rows, -1), q=q.view(rows, -1), k=k.view(rows, -1), v=v.view(rows, -1), xc=xc.view(rows, -1), head=lg)


def _plain_step(b, rows, past_lens, sin, cos, x0, ao):
    from exllamav2_b200 import ext as ext_c
    batch, q_len = _batch(rows)
    new = lambda n: torch.empty((batch, q_len, n), dtype=torch.half, device=DEV)
    xa = x0.clone()
    ext_c.q_attn_forward_2(b.hat[b.style], xa, ao, batch, q_len)
    xa1 = xa.clone().view(rows, -1)
    ext_c.q_mlp_forward_(b.hml, xa.view(rows, -1))
    q, k, v = new(b.heads * b.hd), new(b.kv_heads * b.hd), new(b.kv_heads * b.hd)
    ext_c.q_attn_forward_1(b.hat[b.style], xa, batch, q_len, -1, past_lens, q, k, v, sin, cos)
    xn = ext_c.none_tensor
    lg = torch.empty((rows, 1024), dtype=torch.half, device=DEV)
    xn = torch.empty((rows, b.hidden), dtype=torch.half, device=DEV)
    ext_c.rms_norm(xa.view(rows, -1), b.n3, xn, 1e-5)
    ext_c.gemm_half_q_half(xn, b.lh.q_handle, lg, False)
    return dict(x1=xa1, x2=xa.view(rows, -1), q=q.view(rows, -1), k=k.view(rows, -1), v=v.view(rows, -1), head=lg)


def _inputs(b, rows, seed):
    batch, q_len = _batch(rows)
    rng = np.random.default_rng(seed)
    x0 = torch.from_numpy(rng.normal(0, 1, size=(batch, q_len, b.hidden)).astype(np.float16)).to(DEV)
    ao = torch.from_numpy(rng.normal(0, 1, size=(batch, q_len, b.heads * b.hd)).astype(np.float16)).to(DEV)
    pl = rng.integers(0, 300, size=batch).astype(np.int32)
    pl[0] = 0
    return x0, ao, pl


def _check_step(b, rows, seed):
    batch, q_len = _batch(rows)
    x0, ao, pl_np = _inputs(b, rows, seed)
    pl = torch.from_numpy(pl_np).to(DEV)
    sin_np, cos_np = oracle.rope_tables(b.rot, 512)
    sin, cos = torch.from_numpy(sin_np).to(DEV), torch.from_numpy(cos_np).to(DEV)
    pos = np.repeat(pl_np, q_len) + np.tile(np.arange(q_len), batch)
    got = _chained_step(b, rows, pl, sin, cos, x0, ao)
    plain = _plain_step(b, rows, pl, sin, cos, x0, ao)
    fn = oracle.rope_gptj if b.style == 1 else oracle.rope_neox

    def rope(t, nh):
        return torch.from_numpy(fn(t.cpu().numpy().reshape(rows, nh, b.hd), sin_np, cos_np, pos, b.rot).reshape(rows, -1)).to(DEV)

    xn1 = _t_norm(got["x2"], b.n1)
    truth = {
        "x1": x0.view(rows, -1).double() + ao.view(rows, -1).double() @ b.W["o"] + b.B["o"],
        "x2": _mlp_truth(b, got["x1"]),
        "q": rope((xn1 @ b.W["q"]).half(), b.heads).double(),
        "k": rope((xn1 @ b.W["k"]).half(), b.kv_heads).double(),
        "v": xn1 @ b.W["v"],
        "head": _t_norm(got["xc"], b.n3) @ b.W["a"],
    }
    assert torch.equal(got["xc"], got["x2"]), "the second run's MLP output differs from the first's"
    worst = {}
    for nm, want in truth.items():
        err, e_row, e_plain = _rel(got[nm], want), _row_rel(got[nm], want), _rel(got[nm], plain[nm].double())
        worst[nm] = (err, e_row, e_plain)
        assert err <= 1.5e-3, f"{nm} at {rows} rows: rel-L2 {err:.2e} vs fp64"
        assert e_row <= 4e-3, f"{nm} at {rows} rows: worst row rel-L2 {e_row:.2e} vs fp64"
        assert e_plain <= 2e-3, f"{nm} at {rows} rows: rel-L2 {e_plain:.2e} vs the plain form"
    return worst


@pytest.mark.parametrize("fmt", list(STAGEABLE))
def test_chained_entry_points_every_row_count(fmt):
    b = Block(fmt)
    try:
        for rows in ROWS:
            w = _check_step(b, rows, 100 + rows)
            print(f"WIDE {fmt} rows {rows}: " + " ".join(f"{k} {v[0]:.1e}/{v[1]:.1e}/{v[2]:.1e}" for k, v in w.items()))
    finally:
        b.close()


@pytest.mark.parametrize("variant", ["gelu", "bias", "gelu_bias_gptj"])
def test_epilogue_variants(variant):
    """GELU * up, bias on o_proj and gate / up, GPT-J RoPE, at 17, 33 and 64 rows"""
    b = Block("exl2_54_g128", gelu="gelu" in variant, bias="bias" in variant, rope_style=1 if "gptj" in variant else 2)
    try:
        for rows in (17, 33, 64):
            _check_step(b, rows, 7 * rows)
    finally:
        b.close()


# ---- fused RoPE, bit-exact ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("rot_frac", [1, 2], ids=["full", "partial"])
@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("style", [1, 2], ids=["gptj", "neox"])
def test_fused_rope_bit_exact(style, hd, rot_frac):
    from exllamav2_b200 import ext as ext_c
    heads, kv_heads = 1024 // hd, 256 // hd
    b = Block("exl2_54_g128", heads=heads, kv_heads=kv_heads, hd=hd, rope_style=style, rot=hd // rot_frac)
    fn = oracle.rope_gptj if style == 1 else oracle.rope_neox
    sin_np, cos_np = oracle.rope_tables(b.rot, 512)
    sin, cos = torch.from_numpy(sin_np).to(DEV), torch.from_numpy(cos_np).to(DEV)
    try:
        for rows in (9, 17, 32, 40, 64):
            batch, q_len = _batch(rows)
            x0, ao, pl_np = _inputs(b, rows, rows)
            for mode in ("past_len", "past_lens_only"):
                past_len = 6 if mode == "past_len" else -1
                pl = torch.from_numpy(pl_np).to(DEV)
                base = pl_np + (6 if mode == "past_len" else 0)
                xb = x0.clone()
                ext_c.q_attn_forward_2_ex(b.hat[style], xb, ao, batch, q_len, False, b.chain_mlp)
                ext_c.q_mlp_forward_ex(b.hml, xb.view(rows, -1), True, b.chain_attn)     # q|k|v's inputs, written once
                out = {}
                for nm, st in (("plain", 0), ("fused", style)):
                    q = torch.empty((batch, q_len, heads * hd), dtype=torch.half, device=DEV)
                    k = torch.empty((batch, q_len, kv_heads * hd), dtype=torch.half, device=DEV)
                    v = torch.empty_like(k)
                    ext_c.q_attn_forward_1_ex(b.hat[st], None, batch, q_len, past_len, pl, q, k, v, sin, cos, True)
                    out[nm] = [t.reshape(rows, -1).cpu().numpy() for t in (q, k, v)]
                pos = np.repeat(base, q_len) + np.tile(np.arange(q_len), batch)
                for i, (nh, nm) in enumerate(((heads, "q"), (kv_heads, "k"))):
                    want = fn(out["plain"][i].reshape(rows, nh, hd), sin_np, cos_np, pos, b.rot).reshape(rows, -1)
                    bad = np.count_nonzero(out["fused"][i].view(np.uint16) != want.view(np.uint16))
                    assert bad == 0, f"{nm}: {bad} values differ from the stand-alone rotation ({rows} rows, {mode})"
                assert np.array_equal(out["fused"][2].view(np.uint16), out["plain"][2].view(np.uint16)), "v was rotated"
    finally:
        b.close()


# ---- refusals --------------------------------------------------------------------------------------------------------------------

def _entry_points(b, rows, chain_ok=True):
    from exllamav2_b200 import ext as ext_c
    batch, q_len = _batch(rows) if rows <= 64 else (rows, 1)
    x = torch.randn((batch, q_len, b.hidden), device=DEV).half()
    ao = torch.randn((batch, q_len, b.heads * b.hd), device=DEV).half()
    q = torch.empty((batch, q_len, b.heads * b.hd), dtype=torch.half, device=DEV)
    k = torch.empty((batch, q_len, b.kv_heads * b.hd), dtype=torch.half, device=DEV)
    v = torch.empty_like(k)
    sin_np, cos_np = oracle.rope_tables(b.rot, 512)
    sin, cos = torch.from_numpy(sin_np).to(DEV), torch.from_numpy(cos_np).to(DEV)
    pl = torch.zeros(batch, dtype=torch.int32, device=DEV)
    lg = torch.empty((batch * q_len, 1024), dtype=torch.half, device=DEV)
    return x, [
        ("q_attn_forward_2_ex", lambda: ext_c.q_attn_forward_2_ex(b.hat[b.style], x, ao, batch, q_len, False, b.chain_mlp)),
        ("q_attn_forward_2_ex prepared", lambda: ext_c.q_attn_forward_2_ex(b.hat[b.style], x, ao, batch, q_len, True, None)),
        ("q_mlp_forward_ex", lambda: ext_c.q_mlp_forward_ex(b.hml, x.view(batch * q_len, -1), True, b.chain_attn)),
        ("q_attn_forward_1_ex", lambda: ext_c.q_attn_forward_1_ex(b.hat[b.style], None, batch, q_len, -1, pl, q, k, v, sin, cos, True)),
        ("gemm_half_q_half_prepared", lambda: ext_c.gemm_half_q_half_prepared(b.lh.q_handle, lg, True, 1e-5)),
    ]


def test_65_rows_refused():
    b = Block("exl2_54_g128")
    try:
        x, calls = _entry_points(b, 65)
        before = x.clone()
        for nm, call in calls:
            with pytest.raises(RuntimeError, match="64"):
                call()
            torch.cuda.synchronize()
            assert torch.equal(x, before), f"{nm} modified x"
    finally:
        b.close()


@pytest.mark.parametrize("fmt", ["exl2_4b_g256", "exl2_64_g256_g128", "gptq_nogroup"])
def test_unstageable_groups_refused(fmt):
    b = Block(fmt)
    try:
        for rows in (9, 17, 33, 64):
            x, calls = _entry_points(b, rows)
            before = x.clone()
            for nm, call in calls:
                with pytest.raises(RuntimeError, match="quantisation groups|exl2b_qmatrix_tc_supported"):
                    call()
                torch.cuda.synchronize()
                assert torch.equal(x, before), f"{nm} modified x at {rows} rows"
    finally:
        b.close()


# ---- state: graphs and streams -------------------------------------------------------------------------------------------------

def _mlp_chain(b, x, rows):
    from exllamav2_b200 import ext as ext_c
    batch, q_len = _batch(rows)
    ao = torch.ones((batch, q_len, b.heads * b.hd), dtype=torch.half, device=DEV) * 0.01
    ext_c.q_attn_forward_2_ex(b.hat[b.style], x, ao, batch, q_len, False, b.chain_mlp)
    ext_c.q_mlp_forward_ex(b.hml, x.view(rows, -1), True, b.chain_head)
    lg = torch.empty((rows, 1024), dtype=torch.half, device=DEV)
    ext_c.gemm_half_q_half_prepared(b.lh.q_handle, lg, True, 1e-5)
    return lg


def test_graphs_and_streams():
    from exllamav2_b200 import ext as ext_c
    b = Block("exl2_54_g128")
    try:
        s = torch.cuda.Stream(DEV)
        x8 = torch.randn((8, 1, b.hidden), device=DEV).half()
        x64 = torch.randn((64, 1, b.hidden), device=DEV).half()
        with torch.cuda.stream(s):
            xe = x8.clone()
            eager8 = _mlp_chain(b, xe, 8).clone()          # warm-up: the 8-row buffers and scratch exist before capture
            g8 = torch.cuda.CUDAGraph()
            xg = x8.clone()
            with torch.cuda.graph(g8, stream=s):
                lg8 = _mlp_chain(b, xg, 8)
            xw = x64.clone()
            eager64 = _mlp_chain(b, xw, 64).clone()        # the first wide launch on this stream and these matrices
            ws_wide = ext_c.debug_scratch(DEV, s, "tc_ws_wide")
            assert ws_wide[0] != 0
            xg.copy_(x8)
            g8.replay()
            torch.cuda.synchronize()
            assert torch.equal(lg8, eager8) and torch.equal(xg, xe), "8-row graph captured before the wide launch differs"
            g64 = torch.cuda.CUDAGraph()
            xg64 = x64.clone()
            with torch.cuda.graph(g64, stream=s):
                lg64 = _mlp_chain(b, xg64, 64)
            xg64.copy_(x64)
            g64.replay()
            torch.cuda.synchronize()
            assert torch.equal(lg64, eager64) and torch.equal(xg64, xw), "captured wide step differs from eager"
        s2 = torch.cuda.Stream(DEV)
        with torch.cuda.stream(s2):
            x2 = x64.clone()
            other = _mlp_chain(b, x2, 64).clone()
            torch.cuda.synchronize()
        assert torch.equal(other, eager64)
        for kind in ("tc_ws_wide", "tc_xp_wide"):
            a, c = ext_c.debug_scratch(DEV, s, kind), ext_c.debug_scratch(DEV, s2, kind)
            assert a[0] and c[0] and a[0] != c[0], f"{kind}: streams share wide scratch"
        assert ext_c.debug_scratch(DEV, s, "tc_ws")[0] != ws_wide[0]
    finally:
        b.close()
