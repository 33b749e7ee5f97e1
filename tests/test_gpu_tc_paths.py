"""The 2..16-row path (csrc/gemm_tc.cu, the wgmma dequant-GEMM) against fp64 truth, branch by branch.

This kernel runs every call of 2..16 rows: batched decode and every prompt chunk of the decoder's prefill (8-row chunks with
RoPE fused into the epilogue at per-sequence positions).  Covered here:
  * fused RoPE, GPT-J and NeoX style, full and partial rotary width, per-sequence positions: BIT-EXACT against the
    stand-alone oracle rotation of the same launch's un-rotated output (a rope_style = 0 handle on the same matrices runs the
    identical launch -- same grid, same split-K order -- only the epilogue's rotation mask differs);
  * every row count 2..16 on matrices above the 20 M-weight threshold, so 9..16 rows take two wgmma passes (9: an 8-row pass
    and the one-row tail pass) instead of the dense path, plain and accumulating (residual, strided operands);
  * the 4-bit two-offset form (the tensor core multiplies 1024 + q / 64 + q and the offsets are removed per group afterwards)
    on activation rows that are not zero-mean -- shifted, one-signed, fixed-sign outlier channels, tiny -- next to the dense
    path (no cancellation) and the integer GEMV on the same rows and the same matrix.
Truth: fp64 products over the kernel's own reconstruct(), which test_gpu_linear pins bit-exactly against the oracle.
"""
import math

import numpy as np
import pytest
import torch

import exl2_oracle as oracle
import synth
from test_i8_emulation import quantise_block

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 5e-4


def _lin_np(w_np, K, N):
    from exllamav2_b200.linear import ExLlamaV2Linear, load_tensor_dict
    lin = ExLlamaV2Linear(K, N, has_bias="bias" in w_np, device=DEV)
    lin.load(load_tensor_dict(w_np, DEV))
    return lin


def _lin_dev(K, N, plan, seed, perm_seed=None):
    """plan = (bits, bits_prop, group_size) or ("gptq", group_size, act_order); weights of std ~1/sqrt(K)."""
    from exllamav2_b200 import synthetic
    from exllamav2_b200.linear import ExLlamaV2Linear
    w = synthetic.random_linear(K, N, plan, device=DEV, seed=seed, weight_std=1.0 / math.sqrt(K), perm_seed=perm_seed)
    lin = ExLlamaV2Linear(K, N, device=DEV)
    lin.load(w)
    return lin


def _rel(got: torch.Tensor, want: torch.Tensor) -> float:
    return (torch.linalg.norm(got.double() - want) / torch.linalg.norm(want)).item()


# ---- 1. fused RoPE: bit-exact ------------------------------------------------------------------------------------------------

SHAPES = [(1, 2), (2, 1), (2, 4), (8, 1), (1, 8)]          # (batch, q_len): 2..8 rows, one wgmma pass


def _positions(mode, batch, rng):
    """(past_len, past_lens or None, per-sequence base position)"""
    if mode == "past_len":
        return 6, None, np.full(batch, 6)
    offs = rng.permutation(np.arange(1, 40))[:batch].astype(np.int32)
    if mode == "offsets":
        return 6, offs, 6 + offs
    offs[batch // 2] = 0                                     # past_len = -1: positions from past_lens alone, one of them 0
    return -1, offs, offs.astype(np.int64)


@pytest.mark.parametrize("rot_frac", [1, 2], ids=["full", "partial"])
@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("style", [1, 2], ids=["gptj", "neox"])
def test_fused_rope_bit_exact(style, hd, rot_frac):
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200.ext import none_tensor
    hidden, heads, kv_heads = 512, 8, 2                     # GQA
    rot = hd // rot_frac
    mk = lambda N, s: synth.make_exl2(hidden, N, (5, 4), (0.1, 0.9), 64, seed=s)
    wq, wk, wv = mk(heads * hd, 21), mk(kv_heads * hd, 22), mk(kv_heads * hd, 23)
    wk["q_invperm"], wv["q_invperm"] = wq["q_invperm"].copy(), wq["q_invperm"].copy()
    lq, lk, lv = _lin_np(wq, hidden, heads * hd), _lin_np(wk, hidden, kv_heads * hd), _lin_np(wv, hidden, kv_heads * hd)
    rng = np.random.default_rng(hd * 10 + style + rot_frac)
    nw = torch.from_numpy((1 + 0.1 * rng.normal(size=(hidden,))).astype(np.float16)).to(DEV)
    sin_np, cos_np = oracle.rope_tables(rot, 128)
    sin, cos = torch.from_numpy(sin_np).to(DEV), torch.from_numpy(cos_np).to(DEV)

    def handle(rope_style):
        return ext_c.make_q_attn(nw, none_tensor, True, False, 1e-5, lq.q_handle, lk.q_handle, lv.q_handle, 0,
                                 none_tensor, none_tensor, 64, hidden, heads, kv_heads, hd, 128, True, rope_style, rot,
                                 none_tensor, none_tensor, none_tensor, none_tensor, False, True)
    h0, hr = handle(0), handle(style)
    fn = oracle.rope_gptj if style == 1 else oracle.rope_neox
    for batch, q_len in SHAPES:
        rows = batch * q_len
        x = torch.from_numpy(rng.normal(0, 1, size=(batch, q_len, hidden)).astype(np.float16)).to(DEV)
        for mode in ("past_len", "offsets", "past_lens_only"):
            past_len, offs, base = _positions(mode, batch, rng)
            pl = torch.from_numpy(offs).to(DEV) if offs is not None else none_tensor
            out = {}
            for nm, h in (("plain", h0), ("fused", hr)):
                q = torch.empty((batch, q_len, heads * hd), dtype=torch.half, device=DEV)
                k = torch.empty((batch, q_len, kv_heads * hd), dtype=torch.half, device=DEV)
                v = torch.empty_like(k)
                ext_c.q_attn_forward_1(h, x, batch, q_len, past_len, pl, q, k, v, sin, cos)
                out[nm] = [t.reshape(rows, -1).cpu().numpy() for t in (q, k, v)]
            pos = np.repeat(base, q_len) + np.tile(np.arange(q_len), batch)
            where = f"batch {batch} q_len {q_len} positions {mode}"
            for i, (nh, nm) in enumerate(((heads, "q"), (kv_heads, "k"))):
                want = fn(out["plain"][i].reshape(rows, nh, hd), sin_np, cos_np, pos, rot).reshape(rows, -1)
                got = out["fused"][i]
                bad = np.count_nonzero(got.view(np.uint16) != want.view(np.uint16))
                assert bad == 0, f"{nm}: {bad} values differ from the stand-alone rotation ({where})"
            assert np.array_equal(out["fused"][2].view(np.uint16), out["plain"][2].view(np.uint16)), f"v was touched ({where})"
    for h in (h0, hr):
        ext_c.free_q_attn(h)
    for l in (lq, lk, lv):
        l.unload()


# ---- 4. every row count 2..16, including the two-pass route -------------------------------------------------------------------

BIG = {
    "exl2_54_2048x11008": (2048, 11008, ((5, 4), (0.1, 0.9), 128)),
    "gptq_act_4096x5632": (4096, 5632, ("gptq", 128, True)),
}


@pytest.mark.parametrize("name", list(BIG))
def test_every_row_count(name):
    """M = 2..16 on a matrix above 20 M weights (9..16 rows: two wgmma passes, the second of M - 8 rows; M = 9 is the one-row
    tail pass, which with clear=False adds the residual it loaded before the split-K hand-off).  Plain and accumulating form
    (strided a / c, padding untouched), rel-L2 <= 5e-4 vs fp64, bit-identical on a repeat call."""
    from exllamav2_b200 import ext as ext_c
    K, N, plan = BIG[name]
    lin = _lin_dev(K, N, plan, seed=31)
    W = lin.get_weight_tensor_dq().double()
    g = torch.Generator(device=DEV).manual_seed(7)
    for M in range(2, 17):
        a = torch.randn((M, K), device=DEV, generator=g).half()
        truth = a.double() @ W
        y = lin.forward(a)
        err = _rel(y, truth)
        assert err <= TOL, f"{name} M={M}: rel_l2 {err:.2e}"
        assert torch.equal(y, lin.forward(a)), f"{name} M={M}: repeat call differs"
        c0 = torch.randn((M, N), device=DEV, generator=g).half()
        a_buf = torch.zeros((M, K + 24), dtype=torch.half, device=DEV)
        a_buf[:, :K] = a
        outs = []
        for _ in range(2):
            c_buf = torch.full((M, N + 8), 3.0, dtype=torch.half, device=DEV)
            c_buf[:, :N] = c0
            ext_c.gemm_half_q_half_accum(a_buf[:, :K], lin.q_handle, c_buf[:, :N])
            outs.append(c_buf)
        err = _rel(outs[0][:, :N], truth + c0.double())
        assert err <= TOL, f"{name} M={M} accumulate: rel_l2 {err:.2e}"
        assert bool((outs[0][:, N:] == 3.0).all()), f"{name} M={M}: padding columns written"
        assert torch.equal(outs[0], outs[1]), f"{name} M={M}: accumulate repeat call differs"
    lin.unload()


# ---- 5. activation families across regimes ------------------------------------------------------------------------------------

FAMILIES = ["normal", "mean+2", "mean-3", "abs", "outliers", "tiny"]
MATS = {                                                   # K = 4096, N = 5632: 23 M weights, so 12 rows take two wgmma passes
    "exl2_4": ((4,), (1.0,), 128),
    "gptq": ("gptq", 128, False),
    "gptq_act": ("gptq", 128, True),
    "exl2_32": ((3, 2), (0.5, 0.5), 128),                  # no 4-bit group: the non-offset control
}
REGIMES = (1, 2, 8, 12, 32)                                # integer GEMV, wgmma (one pass), wgmma (two passes), dense


def _family(name, M, K, seed):
    rng = np.random.default_rng(seed)
    z = rng.normal(0, 1, size=(M, K))
    if name == "mean+2":
        z = z + 2
    elif name == "mean-3":
        z = z - 3
    elif name == "abs":
        z = np.abs(z)
    elif name == "outliers":                               # the same channels in every row, each with a fixed sign
        ch = rng.choice(K, size=K // 1024 * 4 + 1, replace=False)
        sign = rng.choice([-1.0, 1.0], size=ch.shape)
        mag = np.full(ch.shape, 64.0)
        mag[0] = 512.0
        z[:, ch] = sign * mag * (1 + np.abs(z[:, ch]))
    elif name == "tiny":
        z = z * 2.0 ** -16                                 # ~1.5e-5: partly fp16-subnormal (< 6.1e-5)
    return z.astype(np.float16)


@pytest.mark.parametrize("mat", list(MATS))
def test_activation_families(mat):
    """rel-L2 vs fp64 per activation family and row regime.  The dense path (M = 32) has no offset cancellation, so the
    wgmma error beside it on the same rows isolates the two-offset form: wgmma <= 2 x dense + 2e-5.  The integer GEMV (one
    row) quantises the row to 16 bits per 128-k block: outlier-free rows are held to 5e-4, rows with outlier channels to the
    quantisation bound of every single output.
    Measured on an H100 (rel-L2 vs fp64): the dense path sits at 2.1e-4 for every family; the wgmma kernel at 2.8e-4 on
    zero-mean rows, and on EXL2 4-bit with shifted or one-signed rows at 3.2e-4 .. 3.9e-4 (1.6 .. 1.9 x dense, where GPTQ 4-bit
    shows 2.3e-4 .. 2.5e-4 and the 3/2-bit control 2.1e-4): the offset cancellation is visible there, inside the contract."""
    K, N = 4096, 5632
    lin = _lin_dev(K, N, MATS[mat], seed=41)
    W = lin.get_weight_tensor_dq().double()
    perm = lin.q_tensors.get("q_perm")
    perm = perm.long() if perm is not None else torch.arange(K, device=DEV)
    report, fails = {}, []
    for fi, fam in enumerate(FAMILIES):
        a = torch.from_numpy(_family(fam, 32, K, 100 + fi)).to(DEV)
        truth = a.double() @ W
        # fp16 output rounding alone: what a correctly rounded result loses (matters only for the tiny family, whose outputs
        # are fp16-subnormal)
        e_round = _rel(truth.half(), truth)
        tol = TOL + 2 * e_round if fam == "tiny" else TOL
        dense = lin.forward(a)
        report[fam] = {}
        for M in REGIMES:
            y = dense[:M] if M == 32 else lin.forward(a[:M].contiguous())
            err, e_dense = _rel(y, truth[:M]), _rel(dense[:M], truth[:M])
            report[fam][M] = err
            where = f"{mat} {fam} M={M}"
            if M == 1 and fam == "outliers":
                # every output within the row-quantisation bound: per 128-k block of the stored row order, half a quantisation
                # step times sum |W| over the block, plus fp16 weight rounding (the kernel applies the scales to exact integer
                # sums), fp32 accumulation and one fp16 output rounding
                ap = a[0][perm].float().cpu().numpy()
                Wp = W[perm].abs()
                bound = torch.zeros((N,), dtype=torch.float64, device=DEV)
                for b in range(K // 128):
                    _, step = quantise_block(ap[b * 128:(b + 1) * 128])
                    bound += 0.5 * float(step) * Wp[b * 128:(b + 1) * 128].sum(0)
                s_abs = a[0].double().abs() @ W.abs()
                bound += (2.0 ** -11 + 2.0 ** -20) * s_abs + truth[0].abs() * 2.0 ** -10 + 2.0 ** -24
                over = (y[0].double() - truth[0]).abs() - bound
                if over.max().item() > 0:
                    fails.append(f"{where}: {int((over > 0).sum())} outputs outside the quantisation bound")
            elif err > tol:
                fails.append(f"{where}: rel_l2 {err:.2e} > {tol:.1e} (dense on the same rows {e_dense:.2e})")
            if M in (2, 8, 12) and err > 2 * e_dense + 2e-5:
                fails.append(f"{where}: wgmma {err:.2e} vs dense {e_dense:.2e} on the same rows")
    print(f"\n{mat}: rel-L2 vs fp64 by family and rows")
    for fam, errs in report.items():
        print(f"  {fam:9s} " + "  ".join(f"M={M}: {e:.2e}" for M, e in errs.items()))
    lin.unload()
    assert not fails, "\n".join(fails)


# ---- 3. chained forms at 2..8 rows vs fp64 --------------------------------------------------------------------------------------

def _t_norm(x: torch.Tensor, w: torch.Tensor, eps=1e-5) -> torch.Tensor:
    xf = x.double()
    return xf * w.double() / torch.sqrt((xf * xf).mean(-1, keepdim=True) + eps)


@pytest.mark.parametrize("batch,q_len", [(1, 2), (5, 1), (2, 4)])
@pytest.mark.parametrize("fmt", ["exl2_54", "gptq_act"])
def test_chained_forms_multi_row(fmt, batch, q_len):
    """The chained decoder step at 2..8 rows: o_proj scatters its output into gate|up's activation buffer with the MLP's norm
    weight and per-strip sums of squares; the MLP (input prepared, 1/rms deferred to after the GEMM) scatters into q|k|v's;
    q|k|v run prepared, with RoPE at per-sequence positions; a second pass chains the MLP into the head instead.  Every
    intermediate is checked against an fp64 composition that starts from the kernel's previous fp16 output (<= 1.5e-3), and
    against the plain forms (<= 2e-3).  Above one row the two forms are not bit-identical: the chained consumer applies 1/rms
    to the fp32 sums after the GEMM, the plain form to the activations before it, so the fp16 roundings fall elsewhere."""
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200.ext import none_tensor
    hidden, inter, heads, hd, vocab = 512, 1408, 8, 64, 1024
    rows = batch * q_len
    if fmt == "exl2_54":
        mk = lambda K, N, s: synth.make_exl2(K, N, (5, 4), (0.1, 0.9), 128, seed=s, scale_max_range=(0.02, 0.08))
        share = "q_invperm"
    else:
        mk = lambda K, N, s: synth.make_gptq(K, N, 128, seed=s, act_order=True)
        share = "g_idx"
    wq, wk, wv, wo = mk(hidden, hidden, 51), mk(hidden, hidden, 52), mk(hidden, hidden, 53), mk(hidden, hidden, 54)
    wk[share], wv[share] = wq[share].copy(), wq[share].copy()
    wg, wu, wd = mk(hidden, inter, 55), mk(hidden, inter, 56), mk(inter, hidden, 57)
    wu[share] = wg[share].copy()
    wh = mk(hidden, vocab, 58)
    lq, lk, lv, lo = (_lin_np(w, hidden, hidden) for w in (wq, wk, wv, wo))
    lg, lu, ld, lh = _lin_np(wg, hidden, inter), _lin_np(wu, hidden, inter), _lin_np(wd, inter, hidden), _lin_np(wh, hidden, vocab)
    Wq, Wk, Wv, Wo, Wg, Wu, Wd, Wh = (l.get_weight_tensor_dq().double() for l in (lq, lk, lv, lo, lg, lu, ld, lh))
    rng = np.random.default_rng(rows * 7 + len(fmt))
    n1, n2, n3 = (torch.from_numpy((1 + 0.1 * rng.normal(size=(hidden,))).astype(np.float16)).to(DEV) for _ in range(3))
    sin_np, cos_np = oracle.rope_tables(hd, 64)
    sin, cos = torch.from_numpy(sin_np).to(DEV), torch.from_numpy(cos_np).to(DEV)
    past_lens_np = rng.permutation(np.arange(0, 40))[:batch].astype(np.int32)
    past_lens = torch.from_numpy(past_lens_np).to(DEV)
    pos = np.repeat(past_lens_np, q_len) + np.tile(np.arange(q_len), batch)
    ta, tb = torch.empty((rows, inter), dtype=torch.half, device=DEV), torch.empty((rows, inter), dtype=torch.half, device=DEV)
    hat = ext_c.make_q_attn(n1, none_tensor, True, False, 1e-5, lq.q_handle, lk.q_handle, lv.q_handle, lo.q_handle,
                            none_tensor, none_tensor, 64, hidden, heads, heads, hd, 64, True, 2, hd,
                            none_tensor, none_tensor, none_tensor, none_tensor, False, True)
    hml = ext_c.make_q_mlp(n2, none_tensor, True, 1e-5, lg.q_handle, lu.q_handle, ld.q_handle, none_tensor, ta, tb, none_tensor,
                           64, False, True, none_tensor, none_tensor, False, True)
    chain_mlp = ext_c.make_chain([lg.q_handle, lu.q_handle], n2)
    chain_attn = ext_c.make_chain([lq.q_handle, lk.q_handle, lv.q_handle], n1)
    chain_head = ext_c.make_chain([lh.q_handle], n3)
    x0 = torch.from_numpy(rng.normal(0, 1, size=(batch, q_len, hidden)).astype(np.float16)).to(DEV)
    ao = torch.from_numpy(rng.normal(0, 1, size=(batch, q_len, hidden)).astype(np.float16)).to(DEV)
    new = lambda n: torch.empty((batch, q_len, n), dtype=torch.half, device=DEV)

    def rope(t):
        return torch.from_numpy(oracle.rope_neox(t.cpu().numpy().reshape(rows, heads, hd), sin_np, cos_np, pos).reshape(rows, -1)).to(DEV)

    def mlp_truth(x):
        xn = _t_norm(x, n2)
        g, u = (xn @ Wg).half().cpu().numpy(), (xn @ Wu).half().cpu().numpy()
        return x.double() + torch.from_numpy(oracle.silu_mul(g, u)).to(DEV).double() @ Wd

    # plain forms
    xa = x0.clone()
    ext_c.q_attn_forward_2(hat, xa, ao, batch, q_len)
    xa1 = xa.clone().view(rows, -1)
    ext_c.q_mlp_forward_(hml, xa.view(rows, -1))
    qa, ka, va = new(hidden), new(hidden), new(hidden)
    ext_c.q_attn_forward_1(hat, xa, batch, q_len, -1, past_lens, qa, ka, va, sin, cos)
    la = torch.empty((rows, vocab), dtype=torch.half, device=DEV)
    ext_c.gemv_norm(xa.view(rows, -1), lh.q_handle, n3, 1e-5, la)

    # chained
    xb = x0.clone()
    ext_c.q_attn_forward_2_ex(hat, xb, ao, batch, q_len, False, chain_mlp)
    xb1 = xb.clone().view(rows, -1)
    ext_c.q_mlp_forward_ex(hml, xb.view(rows, -1), True, chain_attn)
    qb, kb, vb = new(hidden), new(hidden), new(hidden)
    ext_c.q_attn_forward_1_ex(hat, None, batch, q_len, -1, past_lens, qb, kb, vb, sin, cos, True)
    xc = x0.clone()
    ext_c.q_attn_forward_2_ex(hat, xc, ao, batch, q_len, False, chain_mlp)
    ext_c.q_mlp_forward_ex(hml, xc.view(rows, -1), True, chain_head)
    lb = torch.empty((rows, vocab), dtype=torch.half, device=DEV)
    ext_c.gemm_half_q_half_prepared(lh.q_handle, lb, True, 1e-5)

    x2b = xb.view(rows, -1)
    xn1 = _t_norm(x2b, n1)
    checks = [
        ("o_proj + residual", xb1, x0.view(rows, -1).double() + ao.view(rows, -1).double() @ Wo, xa1),
        ("mlp + residual", x2b, mlp_truth(xb1), xa.view(rows, -1)),
        ("q (rope)", qb.view(rows, -1), rope((xn1 @ Wq).half()).double(), qa.view(rows, -1)),
        ("k (rope)", kb.view(rows, -1), rope((xn1 @ Wk).half()).double(), ka.view(rows, -1)),
        ("v", vb.view(rows, -1), xn1 @ Wv, va.view(rows, -1)),
        ("head", lb, _t_norm(xc.view(rows, -1), n3) @ Wh, la),
    ]
    assert torch.equal(xc, xb), "the second run's MLP output differs from the first's"
    for nm, got, truth, plain in checks:
        err, e_plain = _rel(got, truth), _rel(got, plain.double())
        assert err <= 1.5e-3, f"{nm}: rel_l2 {err:.2e} vs fp64"
        assert e_plain <= 2e-3, f"{nm}: rel_l2 {e_plain:.2e} vs the plain form"
    ext_c.free_q_attn(hat)
    ext_c.free_q_mlp(hml)
    for l in (lq, lk, lv, lo, lg, lu, ld, lh):
        l.unload()
