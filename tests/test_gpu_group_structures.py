"""Every group structure the loader accepts, through every block entry point, at every row count, against fp64 truth.

exl2b_qmatrix_create takes EXL2 groups of 32 * 2^n rows with a short last group, and any GPTQ group count, ungrouped
included (one group over all K rows; its nominal size is the next power of two >= K).  The 2..16-row wgmma kernel stages one
group of a 32-column block at a time: at most 128 rows (its activation stage) and 4 KB of weights.  Formats here sit at that
limit (EXL2 8-bit g128: 4096 B), over it (EXL2 4- and 5-bit g256, a 6-bit g256 / 4-bit g128 mix, GPTQ g256 and g512,
ungrouped GPTQ), or stress the group bookkeeping (a short last group of 96 rows, three and five bit widths at different group
sizes).  A matrix over the limit runs on the integer GEMV at one row and on the dense path (reconstruct + GEMM) at every other
row count; before that rule, groups of 256 rows under 4 KB reached the wgmma kernel and overran its activation ring.

Per format:
  * reconstruct() is bit-exact against the numpy oracle, and exl2b_qmatrix_tc_supported says what the rule above says;
  * gemm_half_q_half at 1, 2, 8, 9, 16, 17 and 40 rows, plain and accumulating into a strided c whose padding stays zero,
    <= 5e-4 rel-L2; unit-vector rows return reconstruct()'s weights bit for bit at 1 and 8 rows;
  * q_attn_forward_1 (fused RMSNorm + NeoX RoPE, past_len > 0) and q_attn_forward_2 (residual), q_mlp_forward_ (SiLU and
    GELU), and the tensor-parallel rank's forms -- make_q_attn without o_proj, q_mlp_forward_gateup on a handle made without
    down -- at the same row counts, within the bounds of test_gpu_ops;
  * one row with q/k/v and gate/up on different row permutations (no single integer-GEMV launch for them);
  * the chained forms at 1 and 3 rows against the plain forms, with an 8-bit g128 head; where a format cannot be chained
    above one row the call raises RuntimeError.
Weights: the decoder's synthetic checkpoints (std 1 / sqrt(K)), so block outputs stay O(1) at every bit width.  Truth: fp64
products over the numpy oracle's fp16 weights (equal to the kernel's own reconstruct, checked first).
"""
import math

import numpy as np
import pytest
import torch

import exl2_oracle as oracle

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LIN_TOL = 5e-4          # test_gpu_linear / test_gpu_tc_paths
QKV_TOL = 1.5e-3        # test_gpu_ops.test_q_attn_block: one extra fp16 rounding (norm) + rope roundings
O_TOL = 5e-4            # test_gpu_ops.test_q_attn_block, part 2
MLP_TOL = 3e-3          # test_gpu_ops._q_mlp_block (act(gate) * up and the block output)
ROWS = (1, 2, 8, 9, 16, 17, 40)      # integer GEMV, one and two wgmma passes (9: one-row tail), dense
HEADS, KV_HEADS, HD = 8, 4, 64


# name: (synthetic plan, hidden, intermediate, the wgmma kernel can stage the format's hidden x N matrices)
FORMATS = {
    "exl2_8b_g128": (((8,), (1.0,), 128), 1024, 1536, True),                   # 4096 B: the 8.0 bpw preset / head_bits 8
    "exl2_4b_g256": (((4,), (1.0,), 256), 1024, 1536, False),                  # 4096 B, but 256 rows
    "exl2_5b_g256": (((5,), (1.0,), 256), 1024, 1536, False),
    "exl2_64_g256_g128": (((6, 4), (0.5, 0.5), (256, 128)), 1024, 1536, False),    # one region over, one under
    "exl2_4b_g128_k1376": (((4,), (1.0,), 128), 1376, 1376, True),             # short last group of 96 rows
    "exl2_643_g64_g128_g256": (((6, 4, 3), (0.2, 0.3, 0.5), (64, 128, 256)), 1024, 1536, False),
    "exl2_86542_5regions": (((8, 6, 5, 4, 2), (0.1, 0.1, 0.2, 0.3, 0.3), (32, 64, 32, 128, 64)), 1024, 1536, True),
    "gptq_g256": (("gptq", 256, False), 1024, 1536, False),                    # 4096 B, but 256 rows
    "gptq_g256_act": (("gptq", 256, True), 1024, 1536, False),
    "gptq_g512": (("gptq", 512, False), 1024, 1536, False),
    "gptq_g512_act": (("gptq", 512, True), 1024, 1536, False),
    "gptq_nogroup": (("gptq", -1, True), 1024, 1536, False),                   # desc_act, group_size -1: g_idx all zero
    "gptq_nogroup_no_gidx": (("gptq", -1, False), 1024, 1536, False),          # older checkpoints: no g_idx tensor
    "gptq_nogroup_k1408": (("gptq", -1, True), 1408, 1408, False),             # nominal group 2048 > K
}
OVER = [f for f, v in FORMATS.items() if not v[3]]


def _make(fmt, K, N, seed, perm_seed):
    """synthetic checkpoint tensors on the device (std 1 / sqrt(K)) and a numpy copy for the oracle, taken before loading
    rewrites q_weight and scales q_scale_max in place"""
    from exllamav2_b200 import synthetic
    plan = FORMATS[fmt][0] if fmt in FORMATS else fmt
    w = synthetic.random_linear(K, N, plan, device=DEV, seed=seed, weight_std=1.0 / math.sqrt(K), perm_seed=perm_seed)
    if fmt == "gptq_nogroup_no_gidx":
        del w["g_idx"]
    return w, {k: v.cpu().numpy() for k, v in w.items()}


def _recon(w):
    return oracle.exl2_reconstruct(w) if "q_weight" in w else oracle.gptq_reconstruct(w)


def _staging_ok(w) -> bool:
    """The wgmma kernel's limit restated from the checkpoint tensors: every group's nominal size (EXL2: rows rounded up to
    32 * 2^n; GPTQ: the loader's power-of-two group size) at most 128 rows, and times its bit width at most 1024 (4 KB)."""
    if "q_weight" in w:
        bits, _, rows = oracle.exl2_group_rows(w["q_groups"], w["q_weight"].shape[0], w["q_invperm"].shape[0])
        nominal = [32 * (1 << max(0, math.ceil(math.log2(r // 32)))) for r in rows]
        return all(n <= 128 and n * int(b) <= 1024 for n, b in zip(nominal, bits))
    K = w["qweight"].shape[0] * 8
    return oracle.gptq_groupsize(K, w["qzeros"].shape[0]) <= 128


def _load(w, w_np, K, N):
    """handle + the oracle's fp16 weights on the device; reconstruct() must equal them bit for bit"""
    from exllamav2_b200.linear import ExLlamaV2Linear
    W = _recon(w_np)
    lin = ExLlamaV2Linear(K, N, device=DEV)
    lin.load(w)
    got = lin.get_weight_tensor_dq().cpu().numpy()
    assert np.array_equal(got.view(np.uint16), W.view(np.uint16)), \
        f"reconstruct differs from the oracle in {np.count_nonzero(got.view(np.uint16) != W.view(np.uint16))} weights"
    return lin, torch.from_numpy(W).to(DEV).double()


def _rel(got: torch.Tensor, want: torch.Tensor) -> float:
    return (torch.linalg.norm(got.double() - want) / torch.linalg.norm(want)).item()


def _t_norm(x: torch.Tensor, w: torch.Tensor, eps=1e-5) -> torch.Tensor:
    """oracle.rms_norm on the device: fp64 statistics, y = half(x * w * r)"""
    xf = x.double()
    return (xf * w.double() / torch.sqrt((xf * xf).mean(-1, keepdim=True) + eps)).half()


def _rope(t: torch.Tensor, heads, sin_np, cos_np, pos) -> torch.Tensor:
    rows = t.shape[0]
    r = oracle.rope_neox(t.half().cpu().numpy().reshape(rows, heads, HD), sin_np, cos_np, pos).reshape(rows, -1)
    return torch.from_numpy(r.astype(np.float64)).to(DEV)


def _act(g: torch.Tensor, u: torch.Tensor, gelu: bool) -> torch.Tensor:
    fn = oracle.gelu_mul if gelu else oracle.silu_mul
    return torch.from_numpy(fn(g.half().cpu().numpy(), u.half().cpu().numpy()).astype(np.float64)).to(DEV)


# ---- the matrices of one format ------------------------------------------------------------------------------------------------

class Block:
    """q/k/v/o and gate/up/down of one format (q/k/v and gate/up share their permutation unless own_perm), plus an 8-bit g128
    head, loaded, with their oracle weights."""

    def __init__(self, fmt, own_perm=False):
        _, hid, inter, _ = FORMATS[fmt]
        self.hid, self.inter = hid, inter
        seed = 1000 * (list(FORMATS).index(fmt) + 1) + (500 if own_perm else 0)
        # k / v reuse q's activation order and up reuses gate's (conversion/quantize.py:138-139), unless own_perm
        attn_p, mlp_p = (None, None) if own_perm else (seed + 1, seed + 5)
        shapes = dict(q=(hid, HEADS * HD, attn_p), k=(hid, KV_HEADS * HD, attn_p), v=(hid, KV_HEADS * HD, attn_p),
                      o=(HEADS * HD, hid, None), g=(hid, inter, mlp_p), u=(hid, inter, mlp_p), d=(inter, hid, None))
        self.lin, self.W, self.staging_ok = {}, {}, {}
        for i, (n, (K, N, p)) in enumerate(shapes.items()):
            w, w_np = _make(fmt, K, N, seed + 1 + i, p)
            self.staging_ok[n] = _staging_ok(w_np)
            self.lin[n], self.W[n] = _load(w, w_np, K, N)
        w, w_np = _make(((8,), (1.0,), 128), hid, 1024, seed + 8, None)
        self.staging_ok["h"] = _staging_ok(w_np)
        self.lin["h"], self.W["h"] = _load(w, w_np, hid, 1024)
        rng = np.random.default_rng(seed)
        self.n1, self.n2, self.n3 = (torch.from_numpy((1 + 0.1 * rng.normal(size=(hid,))).astype(np.float16)).to(DEV) for _ in range(3))
        self.sin_np, self.cos_np = oracle.rope_tables(HD, 128)
        self.sin, self.cos = torch.from_numpy(self.sin_np).to(DEV), torch.from_numpy(self.cos_np).to(DEV)
        self.rng = rng
        self.handles = []

    def h(self, n):
        return self.lin[n].q_handle

    def attn(self, with_o=True):
        from exllamav2_b200 import ext as ext_c
        from exllamav2_b200.ext import none_tensor
        a = ext_c.make_q_attn(self.n1, none_tensor, True, False, 1e-5, self.h("q"), self.h("k"), self.h("v"),
                              self.h("o") if with_o else 0, none_tensor, none_tensor, 64, self.hid, HEADS, KV_HEADS, HD, 128,
                              True, 2, HD, none_tensor, none_tensor, none_tensor, none_tensor, False, True)
        self.handles.append(("attn", a))
        return a

    def mlp(self, rows, gelu=False, with_down=True):
        from exllamav2_b200 import ext as ext_c
        from exllamav2_b200.ext import none_tensor
        ta = torch.empty((rows, self.inter), dtype=torch.half, device=DEV)
        tb = torch.empty_like(ta)
        m = ext_c.make_q_mlp(self.n2, none_tensor, True, 1e-5, self.h("g"), self.h("u"), self.h("d") if with_down else 0,
                             none_tensor, ta, tb, none_tensor, 64, gelu, True, none_tensor, none_tensor, False, True)
        self.handles.append(("mlp", m))
        return m, ta

    def x(self, rows, n=None):
        return torch.from_numpy(self.rng.normal(0, 1, size=(rows, n or self.hid)).astype(np.float16)).to(DEV)

    def qkv_truth(self, x, pos):
        xn = _t_norm(x, self.n1).double()
        q, k, v = ((xn @ self.W[n]).half() for n in "qkv")
        return _rope(q, HEADS, self.sin_np, self.cos_np, pos), _rope(k, KV_HEADS, self.sin_np, self.cos_np, pos), v.double()

    def act_truth(self, x, gelu):
        xn = _t_norm(x, self.n2).double()
        return _act(xn @ self.W["g"], xn @ self.W["u"], gelu)

    def close(self):
        from exllamav2_b200 import ext as ext_c
        for kind, hnd in self.handles:
            (ext_c.free_q_attn if kind == "attn" else ext_c.free_q_mlp)(hnd)
        for l in self.lin.values():
            l.unload()


@pytest.fixture(scope="module")
def blocks():
    made = {}

    def get(fmt):
        if fmt not in made:
            for b in made.values():          # one format's matrices on the device at a time
                b.close()
            made.clear()
            made[fmt] = Block(fmt)
        return made[fmt]
    yield get
    for b in made.values():
        b.close()


# ---- the staging rule -------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("fmt", list(FORMATS))
def test_tc_supported_query(fmt, blocks):
    """exl2b_qmatrix_tc_supported agrees with the rule restated from the checkpoint tensors, for every matrix of the block,
    and the format's nominal verdict is the one its name promises."""
    from exllamav2_b200 import ext as ext_c
    b = blocks(fmt)
    for n in "qkvogud":
        assert ext_c.qmatrix_tc_supported(b.h(n)) == b.staging_ok[n], f"{n}_proj"
    assert b.staging_ok["q"] == FORMATS[fmt][3] and b.staging_ok["g"] == FORMATS[fmt][3]
    assert ext_c.qmatrix_tc_supported(b.h("h"))          # 8-bit g128 head: exactly at the limit


# ---- gemm_half_q_half --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("fmt", list(FORMATS))
def test_linear_every_row_count(fmt, blocks):
    from exllamav2_b200 import ext as ext_c
    b = blocks(fmt)
    K, N = b.hid, b.inter
    lin, W = b.lin["g"], b.W["g"]
    g = torch.Generator(device=DEV).manual_seed(11)
    worst = 0.0
    for M in ROWS:
        a = torch.randn((M, K), device=DEV, generator=g).half()
        truth = a.double() @ W
        y = lin.forward(a)
        err = _rel(y, truth)
        worst = max(worst, err)
        assert err <= LIN_TOL, f"M={M}: rel_l2 {err:.2e}"
        c0 = torch.randn((M, N), device=DEV, generator=g).half()
        a_buf = torch.zeros((M, K + 24), dtype=torch.half, device=DEV)
        a_buf[:, :K] = a
        c_buf = torch.zeros((M, N + 8), dtype=torch.half, device=DEV)
        c_buf[:, :N] = c0
        ext_c.gemm_half_q_half_accum(a_buf[:, :K], lin.q_handle, c_buf[:, :N])
        err = _rel(c_buf[:, :N], truth + c0.double())
        worst = max(worst, err)
        assert err <= LIN_TOL, f"M={M} accumulate: rel_l2 {err:.2e}"
        assert torch.count_nonzero(c_buf[:, N:]).item() == 0, f"M={M}: padding columns written"
    for M in (1, 8):                   # integer GEMV; wgmma or, over the staging limit, the dense path
        rows = torch.from_numpy(np.random.default_rng(M).choice(K, size=M, replace=False)).to(DEV)
        e = torch.zeros((M, K), dtype=torch.half, device=DEV)
        e[torch.arange(M, device=DEV), rows] = 1.0
        assert torch.equal(lin.forward(e), W[rows].half()), f"M={M}: unit-vector rows differ from the weights"
    print(f"\n{fmt}: linear worst rel-L2 {worst:.2e}")


def test_linear_ungrouped_down_full_size():
    """Llama-2-7B down projection (K = 11008) as ungrouped act-order GPTQ: one group over all rows, nominal size 16384."""
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200 import synthetic
    from exllamav2_b200.linear import ExLlamaV2Linear
    K, N = 11008, 4096
    w = synthetic.random_gptq(K, N, -1, device=DEV, seed=5, act_order=True, weight_std=1.0 / math.sqrt(K))
    W_np = oracle.gptq_reconstruct({k: v.cpu().numpy() for k, v in w.items()})
    lin = ExLlamaV2Linear(K, N, device=DEV)
    lin.load(w)
    W = lin.get_weight_tensor_dq()
    assert np.array_equal(W.cpu().numpy().view(np.uint16), W_np.view(np.uint16)), "reconstruct differs from the oracle"
    assert not ext_c.qmatrix_tc_supported(lin.q_handle)
    W = W.double()
    g = torch.Generator(device=DEV).manual_seed(12)
    for M in ROWS:
        a = torch.randn((M, K), device=DEV, generator=g).half()
        err = _rel(lin.forward(a), a.double() @ W)
        assert err <= LIN_TOL, f"M={M}: rel_l2 {err:.2e}"
        c0 = torch.randn((M, N), device=DEV, generator=g).half()
        c = c0.clone()
        ext_c.gemm_half_q_half_accum(a, lin.q_handle, c)
        err = _rel(c, a.double() @ W + c0.double())
        assert err <= LIN_TOL, f"M={M} accumulate: rel_l2 {err:.2e}"
    rows = torch.from_numpy(np.random.default_rng(3).choice(K, size=8, replace=False)).to(DEV)
    e = torch.zeros((8, K), dtype=torch.half, device=DEV)
    e[torch.arange(8, device=DEV), rows] = 1.0
    for M in (1, 8):
        assert torch.equal(lin.forward(e[:M]), W[rows[:M]].half()), f"M={M}: unit-vector rows differ from the weights"
    lin.unload()


# ---- attention and MLP blocks ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("fmt", list(FORMATS))
def test_attn_block_every_row_count(fmt, blocks):
    """q_attn_forward_1 (RMSNorm + NeoX RoPE at past_len 7) and q_attn_forward_2 (+ residual) at every row count; the
    tensor-parallel rank's handle (no o_proj) computes part 1 bit for bit like the full one and refuses part 2."""
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200.ext import none_tensor
    b = blocks(fmt)
    full, rank = b.attn(), b.attn(with_o=False)
    past, worst = 7, 0.0
    for rows in ROWS:
        x = b.x(rows)
        outs = []
        for h in (full, rank):
            q = torch.empty((1, rows, HEADS * HD), dtype=torch.half, device=DEV)
            k = torch.empty((1, rows, KV_HEADS * HD), dtype=torch.half, device=DEV)
            v = torch.empty_like(k)
            ext_c.q_attn_forward_1(h, x.view(1, rows, -1), 1, rows, past, none_tensor, q, k, v, b.sin, b.cos)
            outs.append((q.view(rows, -1), k.view(rows, -1), v.view(rows, -1)))
        for t_full, t_rank, nm in zip(*outs, "qkv"):
            assert torch.equal(t_full, t_rank), f"rows {rows}: {nm} of the handle without o_proj differs"
        for got, want, nm in zip(outs[0], b.qkv_truth(x, past + np.arange(rows)), "qkv"):
            err = _rel(got, want)
            worst = max(worst, err)
            assert err <= QKV_TOL, f"rows {rows}: {nm} rel_l2 {err:.2e}"
        ao = b.x(rows, HEADS * HD)
        x2 = x.clone()
        ext_c.q_attn_forward_2(full, x2.view(1, rows, -1), ao.view(1, rows, -1), 1, rows)
        err = _rel(x2, x.double() + ao.double() @ b.W["o"])
        worst = max(worst, err)
        assert err <= O_TOL, f"rows {rows}: o_proj + residual rel_l2 {err:.2e}"
        with pytest.raises(RuntimeError, match="without o_proj"):
            ext_c.q_attn_forward_2(rank, x2.view(1, rows, -1), ao.view(1, rows, -1), 1, rows)
    print(f"\n{fmt}: attention worst rel-L2 {worst:.2e}")


@pytest.mark.parametrize("gelu", [False, True], ids=["silu", "gelu"])
@pytest.mark.parametrize("fmt", list(FORMATS))
def test_mlp_block_every_row_count(fmt, gelu, blocks):
    """q_mlp_forward_ at every row count, and q_mlp_forward_gateup on a handle made without down (act(gate) * up of a
    tensor-parallel rank's slice).  Both pick gate|up's kernel by the same rule: wherever q_mlp_forward_ leaves act(gate) * up
    in temp_a (not fused into the down launch: from 9 rows where the wgmma kernel stages the format, from 2 rows elsewhere),
    q_mlp_forward_gateup leaves the same bits."""
    from exllamav2_b200 import ext as ext_c
    b = blocks(fmt)
    worst = 0.0
    for rows in ROWS:
        x = b.x(rows)
        act = b.act_truth(x, gelu)
        h, ta_full = b.mlp(rows, gelu)
        xt = x.clone()
        ext_c.q_mlp_forward_(h, xt)
        err = _rel(xt, x.double() + act @ b.W["d"])
        worst = max(worst, err)
        assert err <= MLP_TOL, f"rows {rows}: rel_l2 {err:.2e}"
        hr, ta = b.mlp(rows, gelu, with_down=False)
        ext_c.q_mlp_forward_gateup(hr, x, ta)
        err = _rel(ta, act)
        worst = max(worst, err)
        assert err <= MLP_TOL, f"rows {rows}: gate|up rel_l2 {err:.2e}"
        if rows >= (9 if FORMATS[fmt][3] else 2):       # below: act(gate) * up goes to down's operand buffer only
            assert torch.equal(ta, ta_full), f"rows {rows}: gate|up differs from the temp_a of q_mlp_forward_"
        other = b.act_truth(x, not gelu)
        assert _rel(ta, other) > 1e-2, "the other activation fits as well: the test cannot tell them apart"
    print(f"\n{fmt} {'gelu' if gelu else 'silu'}: mlp worst rel-L2 {worst:.2e}")


PERMUTED = [f for f in FORMATS if f.startswith("exl2") or f.endswith("_act")]


@pytest.mark.parametrize("fmt", PERMUTED)
def test_one_row_own_permutations(fmt):
    """One row through blocks whose q/k/v and gate/up were quantised with different activation orders: no single
    integer-GEMV launch serves them, so the blocks take their multi-matrix route at one row."""
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200.ext import none_tensor
    b = Block(fmt, own_perm=True)
    try:
        assert not np.array_equal(b.lin["q"].q_tensors["q_perm"].cpu().numpy(), b.lin["k"].q_tensors["q_perm"].cpu().numpy())
        h = b.attn()
        x = b.x(1)
        q = torch.empty((1, 1, HEADS * HD), dtype=torch.half, device=DEV)
        k = torch.empty((1, 1, KV_HEADS * HD), dtype=torch.half, device=DEV)
        v = torch.empty_like(k)
        ext_c.q_attn_forward_1(h, x.view(1, 1, -1), 1, 1, 5, none_tensor, q, k, v, b.sin, b.cos)
        for got, want, nm in zip((q.view(1, -1), k.view(1, -1), v.view(1, -1)), b.qkv_truth(x, np.array([5])), "qkv"):
            err = _rel(got, want)
            assert err <= QKV_TOL, f"{nm}: rel_l2 {err:.2e}"
        for gelu in (False, True):
            act = b.act_truth(x, gelu)
            m, _ = b.mlp(1, gelu)
            xt = x.clone()
            ext_c.q_mlp_forward_(m, xt)
            err = _rel(xt, x.double() + act @ b.W["d"])
            assert err <= MLP_TOL, f"mlp gelu={gelu}: rel_l2 {err:.2e}"
            mr, ta = b.mlp(1, gelu, with_down=False)
            ext_c.q_mlp_forward_gateup(mr, x, ta)
            err = _rel(ta, act)
            assert err <= MLP_TOL, f"gate|up gelu={gelu}: rel_l2 {err:.2e}"
    finally:
        b.close()


# ---- chained forms ----------------------------------------------------------------------------------------------------------------

def _plain_and_chained(b, rows):
    """One layer step (o_proj, MLP, next q|k|v; a second run feeds the head instead) in the plain and the chained forms.
    Returns {name: (plain, chained)}."""
    from exllamav2_b200 import ext as ext_c
    hat = b.attn()
    hml, _ = b.mlp(rows)
    chain_mlp = ext_c.make_chain([b.h("g"), b.h("u")], b.n2)
    chain_attn = ext_c.make_chain([b.h("q"), b.h("k"), b.h("v")], b.n1)
    chain_head = ext_c.make_chain([b.h("h")], b.n3)
    past = torch.from_numpy(np.arange(3, 3 + rows, dtype=np.int32)).to(DEV)     # one token per sequence, batch = rows
    x0, ao = b.x(rows).view(rows, 1, -1), b.x(rows, HEADS * HD).view(rows, 1, -1)
    new = lambda n: torch.empty((rows, 1, n), dtype=torch.half, device=DEV)

    def head(x, prepared):
        out = torch.empty((rows, 1024), dtype=torch.half, device=DEV)
        if rows == 1:
            ext_c.gemv_norm(x.view(1, -1), b.h("h"), b.n3, 1e-5, out, prepared=prepared)
        elif prepared:
            ext_c.gemm_half_q_half_prepared(b.h("h"), out, True, 1e-5)
        else:
            ext_c.gemv_norm(x.view(rows, -1), b.h("h"), b.n3, 1e-5, out)
        return out

    xa = x0.clone()
    ext_c.q_attn_forward_2(hat, xa, ao, rows, 1)
    xa1 = xa.clone()
    ext_c.q_mlp_forward_(hml, xa.view(rows, -1))
    qa, ka, va = new(HEADS * HD), new(KV_HEADS * HD), new(KV_HEADS * HD)
    ext_c.q_attn_forward_1(hat, xa, rows, 1, -1, past, qa, ka, va, b.sin, b.cos)
    la = head(xa, False)

    xb = x0.clone()
    ext_c.q_attn_forward_2_ex(hat, xb, ao, rows, 1, False, chain_mlp)
    xb1 = xb.clone()
    ext_c.q_mlp_forward_ex(hml, xb.view(rows, -1), True, chain_attn)
    qb, kb, vb = new(HEADS * HD), new(KV_HEADS * HD), new(KV_HEADS * HD)
    ext_c.q_attn_forward_1_ex(hat, None, rows, 1, -1, past, qb, kb, vb, b.sin, b.cos, True)
    xc = x0.clone()
    ext_c.q_attn_forward_2_ex(hat, xc, ao, rows, 1, False, chain_mlp)
    ext_c.q_mlp_forward_ex(hml, xc.view(rows, -1), True, chain_head)
    lb = head(xc, True)
    assert torch.equal(xb, xc), "the second run's MLP output differs from the first's"
    return {"o_proj": (xa1, xb1), "mlp": (xa, xb), "q": (qa, qb), "k": (ka, kb), "v": (va, vb), "head": (la, lb)}


@pytest.mark.parametrize("fmt", list(FORMATS))
def test_chained_one_row_bit_identical(fmt, blocks):
    """At one row every format chains on the integer GEMV: the chained forms read the same fp16 values as the plain forms,
    only from another address, so every output is bit-identical (head: 8-bit g128 through gemv_norm(prepared))."""
    b = blocks(fmt)
    for nm, (plain, chained) in _plain_and_chained(b, 1).items():
        assert torch.equal(plain, chained), f"{nm}: chained form differs from the plain form"


@pytest.mark.parametrize("fmt", [f for f in FORMATS if FORMATS[f][3]])
def test_chained_three_rows(fmt, blocks):
    """At three rows (the wgmma kernel) o_proj reads its own input in both forms and must be bit-identical; a prepared consumer
    (the MLP, q|k|v, the head via gemm_half_q_half_prepared) applies 1/rms after its GEMM instead of before, so it is held to the
    bounds of test_gpu_tc_paths.test_chained_forms_multi_row: <= 1.5e-3 vs an fp64 composition that starts from the chained
    form's previous output, and <= 2e-3 vs the plain form."""
    b = blocks(fmt)
    res = _plain_and_chained(b, 3)
    plain, chained = res["o_proj"]
    assert torch.equal(plain, chained), "o_proj: chained form differs from the plain form"
    x1 = res["o_proj"][1].view(3, -1)
    x = res["mlp"][1].view(3, -1)
    q, k, v = b.qkv_truth(x, np.arange(3, 6))
    truth = {"mlp": x1.double() + b.act_truth(x1, False) @ b.W["d"], "q": q, "k": k, "v": v,
             "head": _t_norm(x, b.n3).double() @ b.W["h"]}
    for nm, want in truth.items():
        plain, chained = res[nm]
        got = chained.view(3, -1)
        err, e_plain = _rel(got, want), _rel(got, plain.view(3, -1).double())
        assert err <= 1.5e-3, f"{nm}: rel_l2 {err:.2e} vs fp64"
        assert e_plain <= 2e-3, f"{nm}: rel_l2 {e_plain:.2e} vs the plain form"


@pytest.mark.parametrize("fmt", OVER)
def test_chained_three_rows_refused(fmt, blocks):
    """Above one row a chained launch needs the wgmma kernel: on a format it cannot stage, every chained entry point raises
    RuntimeError instead of computing something else, and the plain forms still run."""
    from exllamav2_b200 import ext as ext_c
    b = blocks(fmt)
    rows = 3
    hat = b.attn()
    hml, _ = b.mlp(rows)
    chain_mlp = ext_c.make_chain([b.h("g"), b.h("u")], b.n2)
    chain_attn = ext_c.make_chain([b.h("q"), b.h("k"), b.h("v")], b.n1)
    past = torch.zeros((rows,), dtype=torch.int32, device=DEV)
    x, ao = b.x(rows).view(rows, 1, -1), b.x(rows, HEADS * HD).view(rows, 1, -1)
    q, k, v = (torch.empty((rows, 1, n), dtype=torch.half, device=DEV) for n in (HEADS * HD, KV_HEADS * HD, KV_HEADS * HD))
    x0 = x.clone()
    if b.staging_ok["o"]:          # o_proj (K = 512) may fall under the limit where the hidden x N matrices do not
        ext_c.q_attn_forward_2_ex(hat, x.clone(), ao, rows, 1, False, chain_mlp)
    else:
        with pytest.raises(RuntimeError, match="quantisation group"):
            ext_c.q_attn_forward_2_ex(hat, x, ao, rows, 1, False, chain_mlp)
    with pytest.raises(RuntimeError, match="quantisation group"):
        ext_c.q_mlp_forward_ex(hml, x.view(rows, -1), False, chain_attn)
    with pytest.raises(RuntimeError, match="quantisation group"):
        ext_c.q_mlp_forward_ex(hml, x.view(rows, -1), True, None)
    with pytest.raises(RuntimeError, match="quantisation group"):
        ext_c.q_attn_forward_1_ex(hat, None, rows, 1, -1, past, q, k, v, b.sin, b.cos, True)
    assert torch.equal(x, x0), "a refused call modified the residual stream"
    ext_c.q_attn_forward_2(hat, x, ao, rows, 1)
    ext_c.q_mlp_forward_(hml, x.view(rows, -1))
    assert torch.isfinite(x).all()
