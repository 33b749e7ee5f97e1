"""The LoRA launch (csrc/lora.cu) in every regime it takes, against bit-exact invariants and fp64 truth.

tests/lora_regimes.py restates the launch geometry and holds the case lists parametrized here; tests/test_lora_regimes_plan.py
checks on the CPU that together they reach every branch of the kernel: empty and short K slices, 1 / 2 / 4 / 8 warps per column
group with idle warps, the scalar A load (odd ranks, A off 16-byte alignment), the 512-column stage bound with 24 segments, more
than 16 row tiles, output tails on the ADD and ACT_MUL epilogues, partial-width NeoX and GPT-J RoPE, a 112 KB slice per CTA.

Bit-exact: an odd rank gives the bits of the same adapter zero-padded to whole groups of 8 columns (the vector and scalar loads
do the same fmaf sequence per column); A one to seven elements off alignment gives the bits of an aligned copy; B = 0 leaves
q / k / v (RoPE'd by the LoRA launch: rope_kernel's fp16 operations) and the O output bit-identical to the call without
adapters, and the MLP output too where that call runs act_mul_kernel (the dense path); B changed in place is seen by a graph
captured before the change.

fp64: test_gpu_lora.Blocks' truth, with partial rotary widths, blocks without a layernorm or a residual.  Besides 1e-3 rel-L2
over each tensor, every row (and every head of q / k / v) within ROW_TOL / HEAD_TOL, so one wrong row tile, cluster or head cannot
hide in a large tensor.  "Dominant" adapters scale B so that the delta is ~3x the base output on q / k / v, o and down; the
bound then measures the LoRA arithmetic rather than the base GEMM (gate / up keep ~20 %: act(gate) * up must stay in fp16 range).
"""
import math

import numpy as np
import pytest
import torch

import lora_regimes as lr
import synth
import decoder_truth as dt
import test_gpu_decoder_lora as tdl
import test_gpu_full_shapes as tfs
import test_gpu_group_structures as tgs
from test_gpu_lora import ATTN, EPS, MLP, Blocks, _f64

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-3            # whole tensor, as test_gpu_lora
ROW_TOL = 4e-3        # each row
HEAD_TOL = 3e-3       # each head of q / k / v over all rows
POSITIONS = 1152      # sin / cos rows: every position a case uses
WORST = {"tensor": (0.0, ""), "row": (0.0, ""), "head": (0.0, "")}      # the largest error of each kind and its case


class Rig(Blocks):
    """test_gpu_lora.Blocks over one of lora_regimes.BLOCKS (synthetic EXL2 5/4-bit g64), a group format of
    test_gpu_group_structures ("fmt:<name>") or the 70B layer of test_gpu_full_shapes, with attention handles per RoPE style and
    rotary width, and optionally without the blocks' layernorm or residual."""

    def __init__(self, block, norm=True, has_residual=True, own_perm=False):
        from exllamav2_b200 import ext
        from exllamav2_b200.ext import none_tensor
        hid, H, KVH, hd, inter, style, rot = lr.block_shape(block)
        self.hidden, self.heads, self.kvh, self.hd, self.inter = hid, H, KVH, hd, inter
        self.gelu, self.bias, self.adapters = False, {}, {}
        self.use_norm, self.has_residual = norm, has_residual
        self.src = None
        if block.startswith("fmt:"):
            self.src = tgs.Block(block[4:], own_perm=own_perm)
            self.lins = dict(zip(ATTN + MLP, (self.src.lin[n] for n in "qkvogud")))
            self.W = dict(zip(ATTN + MLP, (self.src.W[n] for n in "qkvogud")))
            self.stageable = all(self.src.staging_ok[n] for n in "qkvogud")
        elif block == "70b":
            self.src = tfs.Block70()
            self.lins = dict(zip(ATTN + MLP, (self.src.lin[n] for n in "qkvogud")))
            self.W = {k: _f64(l.get_weight_tensor_dq()) for k, l in self.lins.items()}
            self.stageable = True
        else:
            mk = lambda K, N, s, sm=(0.5, 4.0): synth.make_exl2(K, N, (5, 4), (0.1, 0.9), 64, seed=10 * hid + s, scale_max_range=sm)
            ws = [mk(hid, H * hd, 1), mk(hid, KVH * hd, 2), mk(hid, KVH * hd, 3), mk(H * hd, hid, 4)]
            ws[1]["q_invperm"], ws[2]["q_invperm"] = ws[0]["q_invperm"].copy(), ws[0]["q_invperm"].copy()
            sm = (0.02, 0.08)
            ws += [mk(hid, inter, 5, sm), mk(hid, inter, 6, sm), mk(inter, hid, 7, sm)]
            ws[5]["q_invperm"] = ws[4]["q_invperm"].copy()
            from test_gpu_lora import _lin
            shapes = [(hid, H * hd), (hid, KVH * hd), (hid, KVH * hd), (H * hd, hid), (hid, inter), (hid, inter), (inter, hid)]
            self.lins = {n: _lin(w, K, N) for n, w, (K, N) in zip(ATTN + MLP, ws, shapes)}
            self.W = {k: _f64(l.get_weight_tensor_dq()) for k, l in self.lins.items()}
            self.stageable = True
        rng = np.random.default_rng(hid + 7)
        self.n1 = torch.from_numpy((1 + 0.1 * rng.normal(size=(hid,))).astype(np.float16)).to(DEV)
        self.n2 = torch.from_numpy((1 + 0.1 * rng.normal(size=(hid,))).astype(np.float16)).to(DEV)
        self.ta = torch.empty((64, inter), dtype=torch.half, device=DEV)
        self.tb = torch.empty_like(self.ta)
        L = self.lins
        self.handles = {}
        self.use(style, rot)
        self.mlp = ext.make_q_mlp(self.n2 if norm else none_tensor, none_tensor, True, EPS, L["gate_proj"].q_handle,
                                  L["up_proj"].q_handle, L["down_proj"].q_handle, none_tensor, self.ta, self.tb, none_tensor, 64,
                                  False, has_residual, none_tensor, none_tensor, False, True)

    def use(self, style, rot):
        """the attention handle (made on first use) and sin / cos tables for RoPE `style` over the first `rot` features"""
        from exllamav2_b200 import ext
        from exllamav2_b200.ext import none_tensor
        if (style, rot) not in self.handles:
            L = self.lins
            h = ext.make_q_attn(self.n1 if self.use_norm else none_tensor, none_tensor, True, False, EPS, L["q_proj"].q_handle,
                                L["k_proj"].q_handle, L["v_proj"].q_handle, L["o_proj"].q_handle, none_tensor, none_tensor, 64,
                                self.hidden, self.heads, self.kvh, self.hd, POSITIONS, self.has_residual, style, rot, none_tensor,
                                none_tensor, none_tensor, none_tensor, False, True)
            ang = np.arange(POSITIONS)[:, None] * (1.0 / 10000 ** (np.arange(0, rot, 2) / rot))[None, :]
            ang = np.concatenate([ang, ang], -1) if style == lr.NEOX else np.repeat(ang, 2, axis=-1)
            self.handles[(style, rot)] = (h, torch.from_numpy(np.sin(ang).astype(np.float16)).to(DEV),
                                          torch.from_numpy(np.cos(ang).astype(np.float16)).to(DEV))
        self.attn, self.sin, self.cos = self.handles[(style, rot)]
        self.rope_style, self.rot = style, rot

    # ---- truth: partial rotary, no layernorm, no residual ----
    def norm(self, x, w):
        return super().norm(x, w) if self.use_norm else _f64(x)

    def rope(self, t, heads, pos):
        S = self.rot
        t = t.reshape(-1, heads, self.hd).clone()
        c, s = _f64(self.cos)[pos][:, None, :], _f64(self.sin)[pos][:, None, :]
        r = t[..., :S].clone()
        if self.rope_style == lr.NEOX:
            h = S // 2
            l, rr = r[..., :h], r[..., h:]
            t[..., :S] = torch.cat([l * c[..., :h] - rr * s[..., :h], rr * c[..., :h] + l * s[..., :h]], -1)
        else:
            x0, x1 = r[..., 0::2], r[..., 1::2]
            t[..., 0:S:2] = x0 * c[..., 0::2] - x1 * s[..., 0::2]
            t[..., 1:S:2] = x1 * c[..., 1::2] + x0 * s[..., 1::2]
        return t.view(t.shape[0], -1)

    def truth_attn2(self, x, ao, loras):
        y = super().truth_attn2(x, ao, loras)
        return y if self.has_residual else y - _f64(x).view(-1, self.hidden)

    def truth_mlp(self, x, loras):
        y = super().truth_mlp(x, loras)
        return y if self.has_residual else y - _f64(x).view(-1, self.hidden)

    def free(self):
        from exllamav2_b200 import ext
        for h, _, _ in self.handles.values():
            ext.free_q_attn(h)
        ext.free_q_mlp(self.mlp)
        if self.src is not None:
            self.src.close()
        else:
            for l in self.lins.values():
                l.unload()
        self.W = {}


_RIGS = {}
_BIG = ("fmt:", "70b")          # one of these on the device at a time


def rig(block, **kw):
    key = (block, tuple(sorted(kw.items())))
    if key not in _RIGS:
        if block.startswith(_BIG):
            for k in [k for k in _RIGS if k[0].startswith(_BIG)]:
                _RIGS.pop(k).free()
            torch.cuda.empty_cache()
        _RIGS[key] = Rig(block, **kw)
    return _RIGS[key]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nLORA REGIMES worst rel-L2: " + "  ".join(f"{k} {e:.3e} ({n})" for k, (e, n) in WORST.items()))
    for r in _RIGS.values():
        r.free()
    _RIGS.clear()


def adapters(r, spec, seed=0, dominant=False, zero_b=False):
    """spec [(id, {projection: rank})] -> {id: {projection: (A, B)}}: A ~ N(0, 1/K); B sized so the delta is ~20 % of the
    projection's output, or (dominant) ~3x it on q / k / v, o and down"""
    out = {}
    for key, ranks in spec:
        g = torch.Generator(device=DEV).manual_seed(1000 * seed + key)
        ad = {}
        for t, rank in ranks.items():
            K, N = r.shape(t)
            frac = 3.0 if dominant and t not in ("gate_proj", "up_proj") else 0.2
            a = (torch.randn((K, rank), device=DEV, generator=g) / math.sqrt(K)).half()
            b = (torch.randn((rank, N), device=DEV, generator=g) * (frac * math.sqrt(K) * r.W[t].std().item() / math.sqrt(rank))).half()
            ad[t] = (a, b.zero_() if zero_b else b)
        out[key] = ad
    return out


def _note(kind, err, name):
    if err > WORST[kind][0]:
        WORST[kind] = (err, name)


def check(name, got, want, heads=None, tol=TOL):
    """rel-L2 over the tensor, per row, and per head (heads: q / k / v laid out [rows, heads * hd])"""
    g = _f64(got).reshape(want.shape)
    d = g - want
    err = (d.norm() / want.norm()).item()
    row = (d.norm(dim=-1) / want.norm(dim=-1)).max().item()
    _note("tensor", err, name)
    _note("row", row, name)
    assert err <= tol, f"{name}: rel-L2 {err:.2e}"
    assert row <= ROW_TOL, f"{name}: worst row rel-L2 {row:.2e} (row {int((d.norm(dim=-1) / want.norm(dim=-1)).argmax())})"
    if heads:
        dh, wh = d.view(d.shape[0], heads, -1), want.view(d.shape[0], heads, -1)
        per = dh.pow(2).sum((0, 2)).sqrt() / wh.pow(2).sum((0, 2)).sqrt()
        _note("head", per.max().item(), name)
        assert per.max().item() <= HEAD_TOL, f"{name}: head {int(per.argmax())} rel-L2 {per.max().item():.2e}"


def split(rows):
    return (2, rows // 2) if rows % 2 == 0 and rows > 1 else (1, rows)


def inputs(r, rows, seed):
    rng = np.random.default_rng(seed)
    x = torch.from_numpy(rng.normal(0, 1, size=(rows, r.hidden)).astype(np.float16)).to(DEV)
    ao = torch.from_numpy(rng.normal(0, 1, size=(rows, r.heads * r.hd)).astype(np.float16)).to(DEV)
    return x, ao


_PLENS = {}


def plens(B):
    """past_lens 5 + 17 b (made before any capture)"""
    if B not in _PLENS:
        _PLENS[B] = torch.tensor([5 + 17 * b for b in range(B)], dtype=torch.int32, device=DEV)
    return _PLENS[B]


def positions(B, T, past=-1):
    """each row's RoPE position as the kernels take it: past_len -1 reads past_lens, past_len >= 0 adds it"""
    base = np.array([5 + 17 * b for b in range(B)]) + (0 if past == -1 else past)
    return torch.as_tensor(np.concatenate([base[b] + np.arange(T) for b in range(B)]), device=DEV)


def run(r, x, ao, loras, B, T, past=-1):
    """q, k, v, the O output and the MLP output of one pass"""
    q, k, v = r.attn1(x.view(B, T, -1), B, T, past, loras, plens(B))
    o = r.attn2(x.view(B, T, -1), ao.view(B, T, -1), B, T, loras)
    return q, k, v, o, r.mlp_fwd(x, loras)


def check_all(r, x, ao, loras, B, T, name, past=-1):
    q, k, v, o, m = run(r, x, ao, loras, B, T, past)
    tq, tk, tv = r.truth_attn1(x, positions(B, T, past), loras)
    check(f"{name} q", q, tq, r.heads)
    check(f"{name} k", k, tk, r.kvh)
    check(f"{name} v", v, tv, r.kvh)
    check(f"{name} o", o, r.truth_attn2(x, ao, loras))
    check(f"{name} mlp", m, r.truth_mlp(x, loras))


def bits_equal(a, b, name):
    n = int((a.view(torch.int16) != b.view(torch.int16)).sum())
    assert n == 0, f"{name}: {n} of {a.numel()} values differ"


def ids_of(spec):
    return [k for k, _ in spec]


# ---- a. bit-exact invariants ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("rank,rows", lr.PADDED_CASES)
def test_odd_rank_equals_padded(rank, rows):
    """rank r on every projection == the same A / B with zero columns / rows up to rank_slots(r), bit for bit on all four
    stages; the odd form also within the fp64 bounds"""
    r = rig("hd64")
    r.use(lr.NEOX, 64)
    odd = adapters(r, lr.uniform(rank), seed=rank)
    s = lr.rank_slots(rank)
    pad = {k: {t: (torch.nn.functional.pad(a, (0, s - rank)).contiguous(), torch.nn.functional.pad(b, (0, 0, 0, s - rank)).contiguous())
               for t, (a, b) in ad.items()} for k, ad in odd.items()}
    x, ao = inputs(r, rows, rows + rank)
    B, T = split(rows)
    r.set(pad)
    want = run(r, x, ao, [1], B, T)
    want = [t.clone() for t in want]
    r.set(odd)
    got = run(r, x, ao, [1], B, T)
    for g, w, n in zip(got, want, ("q", "k", "v", "o", "mlp")):
        bits_equal(g, w, f"rank {rank} {n}")
    check_all(r, x, ao, [1], B, T, f"rank {rank} rows {rows}")


@pytest.mark.parametrize("offset,rows", lr.MISALIGNED_CASES)
def test_misaligned_a_equals_aligned(offset, rows):
    """A as a contiguous view `offset` elements into a larger buffer (data_ptr % 16 != 0: the scalar load) == an aligned copy"""
    r = rig("hd64")
    r.use(lr.NEOX, 64)
    al = adapters(r, lr.uniform(16), seed=offset)
    mis = {}
    for k, ad in al.items():
        mis[k] = {}
        for t, (a, b) in ad.items():
            buf = torch.zeros(a.numel() + 8, dtype=torch.half, device=DEV)
            v = buf[offset:offset + a.numel()].view(a.shape)
            v.copy_(a)
            assert v.is_contiguous() and v.data_ptr() % 16 != 0
            mis[k][t] = (v, b)
    x, ao = inputs(r, rows, rows + 31)
    B, T = split(rows)
    r.set(al)
    want = [t.clone() for t in run(r, x, ao, [1], B, T)]
    r.set(mis)
    got = run(r, x, ao, [1], B, T)
    for g, w, n in zip(got, want, ("q", "k", "v", "o", "mlp")):
        bits_equal(g, w, f"offset {offset} {n}")


@pytest.mark.parametrize("block,style,rot,rows,past", lr.ZERO_B_CASES)
def test_zero_b_bit_identical(block, style, rot, rows, past):
    """B = 0 on every projection at odd ranks: q / k / v and the O output carry the bits of the call without adapters; the MLP
    output too where the call without adapters forms act(gate) * up in act_mul_kernel's fp16 operations -- the dense path, and
    one row, where the down launch's prologue does (gemv_i8.cuh I8_SILU_MUL) -- elsewhere (the wgmma epilogue) it is held to the
    fp64 bound"""
    r = rig(block)
    r.use(style, rot)
    r.set(adapters(r, lr.ODD, zero_b=True))
    x, ao = inputs(r, rows, rows + rot)
    B, T = split(rows)
    got = run(r, x, ao, [2, 1], B, T, past)
    got = [t.clone() for t in got]
    want = run(r, x, ao, [], B, T, past)
    for g, w, n in zip(got[:4], want[:4], ("q", "k", "v", "o")):
        bits_equal(g, w, n)
    if rows == 1 or rows > 16 or not r.stageable:
        bits_equal(got[4], want[4], "mlp")
    else:
        check("mlp", got[4], r.truth_mlp(x, [1, 2]))
    tq, tk, _ = r.truth_attn1(x, positions(B, T, past), [])
    check("q", got[0], tq, r.heads)
    check("k", got[1], tk, r.kvh)


@pytest.mark.parametrize("rows", [1, 8, 40])
def test_inplace_b_seen_by_captured_graph(rows):
    """B changed in place after capture: the replay equals an eager call with the new B (the adapter list travels by value,
    A and B by address)"""
    r = rig("hd64")
    r.use(lr.NEOX, 64)
    ads = adapters(r, lr.ODD, seed=5)
    r.set(ads)
    x, ao = inputs(r, rows, rows + 41)
    B, T = split(rows)
    loras = [1, 2]
    run(r, x, ao, loras, B, T)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        run(r, x, ao, loras, B, T)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            outs = run(r, x, ao, loras, B, T)
    torch.cuda.synchronize()
    for ad in ads.values():
        for a, b in ad.values():
            b.mul_(-0.5)
    g.replay()
    torch.cuda.synchronize()
    replayed = [t.clone() for t in outs]
    eager = run(r, x, ao, loras, B, T)
    for a, b, n in zip(replayed, eager, ("q", "k", "v", "o", "mlp")):
        bits_equal(a, b, n)
    check_all(r, x, ao, loras, B, T, "new B")


# ---- b. fp64 truth per regime ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("fmt,rows,which", lr.FORMAT_CASES)
def test_formats(fmt, rows, which):
    """every group format under adapted stages: the integer GEMV, the wgmma kernel and the dense path as the base"""
    r = rig("fmt:" + fmt)
    spec = lr.ODD if which == "odd" else lr.DOWN_ONLY
    r.set(adapters(r, spec, seed=rows))
    x, ao = inputs(r, rows, rows + 3)
    check_all(r, x, ao, ids_of(spec)[::-1], *split(rows), f"{fmt} {which} rows {rows}")


@pytest.mark.parametrize("fmt", lr.OWN_PERM_CASES)
def test_formats_own_permutations(fmt):
    """one row with q / k / v and gate / up on different permutations (no single integer-GEMV launch for them)"""
    r = rig("fmt:" + fmt, own_perm=True)
    r.set(adapters(r, lr.ODD, seed=77))
    x, ao = inputs(r, 1, 77)
    check_all(r, x, ao, [1, 2], 1, 1, f"{fmt} own permutations")


@pytest.mark.parametrize("dominant", [False, True])
@pytest.mark.parametrize("block,rows", lr.GEOMETRY_CASES)
def test_geometry(block, rows, dominant):
    """empty and short K slices, N tails on gate|up and down, head dims 80 / 96 / 256 with partial rotary widths"""
    r = rig(block)
    r.use(*lr.block_shape(block)[5:])
    r.set(adapters(r, lr.ODD, seed=rows, dominant=dominant))
    x, ao = inputs(r, rows, rows + 13)
    check_all(r, x, ao, [1, 2], *split(rows), f"{block} rows {rows}", past=3 if rows % 2 else -1)


@pytest.mark.parametrize("stage,R,rows", lr.STACK_CASES)
def test_stacked_widths(stage, R, rows):
    """R stacked columns on one stage (1 to 64 column groups, the bound 512 with 24 segments on q|k|v), forwarded with the ids
    in reverse registration order and one registered nowhere"""
    r = rig("hd64")
    r.use(lr.NEOX, 64)
    spec = lr.stacked(stage, R)
    if len(spec) < 8:
        spec = spec + [(99, {p: 8 for p in lr.STAGES[stage]})]        # registered, not forwarded
    r.set(adapters(r, spec, seed=R, dominant=True))
    loras = [k for k, _ in lr.stacked(stage, R)][::-1] + [999]
    x, ao = inputs(r, rows, rows + R)
    check_all(r, x, ao, loras, *split(rows), f"{stage} R {R} rows {rows}")


@pytest.mark.parametrize("rows,seqs", lr.LONG_ROWS)
def test_long_prompts(rows, seqs):
    """129 / 256 / 1000 rows of several sequences: past 16 row tiles each tile has one cluster that splits every output unit"""
    r = rig("hd64")
    r.use(lr.NEOX, 64)
    r.set(adapters(r, lr.ODD, seed=rows, dominant=True))
    x, ao = inputs(r, rows, rows)
    check_all(r, x, ao, [1, 2], seqs, rows // seqs, f"{rows} rows")


@pytest.mark.parametrize("rows", lr.FULL_ROWS)
def test_llama70b_layer(rows):
    """one 70B-shaped layer: down stages 112 KB of fp32 input rows per CTA at 8 rows"""
    r = rig("70b")
    r.use(lr.NEOX, 128)
    r.set(adapters(r, lr.uniform(16), seed=rows))
    x, ao = inputs(r, rows, rows + 70)
    check_all(r, x, ao, [1], 1, rows, f"70b rows {rows}", past=11)


@pytest.mark.parametrize("opt,rows", lr.OPTION_CASES)
def test_block_options(opt, rows):
    """blocks made without a layernorm (the LoRA launch's 1/rms is 1), and without the residual (o and down overwrite x)"""
    r = rig("hd64", norm=opt != "no_norm", has_residual=opt != "no_residual")
    r.use(lr.NEOX, 64)
    r.set(adapters(r, lr.ODD, seed=rows, dominant=True))
    x, ao = inputs(r, rows, rows + 5)
    check_all(r, x, ao, [1, 2], *split(rows), f"{opt} rows {rows}")


# ---- c. the decoder ------------------------------------------------------------------------------------------------------------

STAGE_TOL = 3e-3      # each stage of a decode step against fp64 on its own inputs
LAYER_TOL = 6e-3      # each layer of a decode step against the exact layer on the decoder's own input to it
# The decode steps after the 2 x 96 prompt on the head-dim-128 model meet an input whose output is ill-conditioned: at the second
# step (position 97) sequence 1 sat 2.3e-2 from the exact forward, 6.0x its fp16 floor (3.9e-3), over D6's bound (1.3e-2).  Every
# stage of that step -- q / k / v with the LoRA launch, attention, o, the MLP -- was within 1.1e-3 of fp64 on its own inputs, layer
# 0's output 1.9e-3 from exact (as at every other step), and the EXACT layer 1 started from that output already 2.2e-2 from the
# exact forward: the model itself multiplies a 1.9e-3 departure by 11 there.  So each step is checked stage by stage and layer by
# layer, where the bounds are tight, and end to end at 8x the floor where the floor dominates (D6's 1e-2 elsewhere).
DECODE_FLOOR_RATIO = 8.0
_STAGES = ("q_attn_forward_1", "paged_attn_decode_q4", "q_attn_forward_2", "q_mlp_forward_")


def _decode_traced(dec, ids, monkeypatch):
    """dec.decode(ids), recording every block call of the step: (name, arguments before, arguments after), tensors cloned"""
    from exllamav2_b200 import ext
    calls = []

    def spy(name, fn):
        def f(*a, **kw):
            before = [t.clone() if isinstance(t, torch.Tensor) else t for t in a]
            fn(*a, **kw)
            calls.append((name, before, [t.clone() if isinstance(t, torch.Tensor) else t for t in a]))
        return f

    with monkeypatch.context() as m:
        for name in _STAGES:
            m.setattr(ext, name, spy(name, getattr(ext, name)))
        out = dec.decode(torch.from_numpy(ids).to(DEV)).float().cpu().numpy()
        torch.cuda.synchronize()
    assert [c[0] for c in calls] == list(_STAGES) * dec.cfg.num_layers
    return out, calls


def _check_decode_stages(dec, truth, ids, calls, post):
    """each stage of each layer against fp64 on the decoder's own inputs to it, and each layer against the exact layer on the
    decoder's own input to it"""
    from exl2_oracle import rel_l2
    cfg = dec.cfg
    H, KVH, hd = cfg.num_heads, cfg.num_kv_heads, cfg.head_dim
    row = lambda t, b: t.float().cpu().numpy().astype(np.float64).reshape(ids.shape[0], -1)[b:b + 1]
    worst = {}
    for b in range(ids.shape[0]):
        start = int(post["seqlens"][b]) - 1
        pos = np.array([start])
        for li, L in enumerate(truth.layers):
            (_, f1, f1o), (_, _, ato), (_, f2, f2o), (_, m, mo) = calls[4 * li:4 * li + 4]
            pk, pv = dt.cache_kv(post, cfg, dec.cache.wbits, li, b, 0, start)
            d = lambda p, inp: truth._d(li, p, inp)

            def qkv(x):
                xn = dt.rms_norm(x, L.input_norm, truth.eps)
                return (dt.rope_neox((xn @ L.wq + d("q_proj", xn)).reshape(1, H, hd), truth.sin, truth.cos, pos),
                        dt.rope_neox((xn @ L.wk + d("k_proj", xn)).reshape(1, KVH, hd), truth.sin, truth.cos, pos),
                        (xn @ L.wv + d("v_proj", xn)).reshape(1, KVH, hd))

            def attn(q, k, v):
                return dt.attention(q, np.concatenate([pk, k]), np.concatenate([pv, v]), start).reshape(1, -1)

            def o_proj(x, ao):
                return x + ao @ L.wo + d("o_proj", ao)

            def mlp(x):
                xn = dt.rms_norm(x, L.post_norm, truth.eps)
                a = dt.silu(xn @ L.wg + d("gate_proj", xn)) * (xn @ L.wu + d("up_proj", xn))
                return x + a @ L.wd + d("down_proj", a)

            x_in = row(f1[1], b)
            got_qkv = [row(f1o[i], b) for i in (6, 7, 8)]
            want_qkv = qkv(x_in)
            errs = {n: rel_l2(g.reshape(-1), w.reshape(-1)) for n, g, w in zip("qkv", got_qkv, want_qkv)}
            q, k, v = (g.reshape(1, -1, hd) for g in got_qkv)
            errs["attn"] = rel_l2(row(ato[9], b).reshape(-1), attn(q, k, v).reshape(-1))
            errs["o"] = rel_l2(row(f2o[1], b).reshape(-1), o_proj(row(f2[1], b), row(f2[2], b)).reshape(-1))
            errs["mlp"] = rel_l2(row(mo[1], b).reshape(-1), mlp(row(m[1], b)).reshape(-1))
            for n, e in errs.items():
                worst[n] = max(worst.get(n, 0.0), e)
                assert e <= STAGE_TOL, f"seq {b} layer {li} {n}: rel-L2 {e:.2e} against fp64 on its own inputs"
            x = x_in
            y = mlp(o_proj(x, attn(*qkv(x))))
            e = rel_l2(row(mo[1], b).reshape(-1), y.reshape(-1))
            worst["layer"] = max(worst.get("layer", 0.0), e)
            assert e <= LAYER_TOL, f"seq {b} layer {li}: rel-L2 {e:.2e} against the exact layer on its own input"
    return worst


@pytest.mark.parametrize("cache_attn", [False, True])
def test_decoder_long_prefill_rows(cache_attn, monkeypatch):
    """prefill_rows at 2 x 96 rows (24 row tiles) with odd-rank adapters, then decode steps, teacher-forced against fp64: end to
    end, layer by layer and stage by stage"""
    from exllamav2_b200.model import ExLlamaV2Decoder
    dec = ExLlamaV2Decoder(tdl._cfg("hd128" if cache_attn else "small"), device=DEV, seed=tdl.SEED, batch_size=2, cache_len=512,
                           cache_bits=4)
    (r0, t0), (r1, t1) = lr.DECODER_ADAPTERS
    dec.set_loras([dec.load_lora(r0, targets=t0, seed=1), dec.load_lora(r1, targets=t1, scaling=0.5, seed=2)])
    truth = tdl._truth(dec)
    V = dec.cfg.vocab_size
    tdl._check(dec, truth, "P3", "rows", tdl._ids(2, lr.DECODER_ROWS // 2, V, 80),
               lambda x: dec.prefill_rows(x, cache_attn=cache_attn))
    for s in range(3):
        ids = tdl._ids(2, 1, V, 81 + s)
        pre = dt.snapshot(dec)
        out, calls = _decode_traced(dec, ids, monkeypatch)
        post = dt.snapshot(dec)
        worst = _check_decode_stages(dec, truth, ids, calls, post)
        err, floor, _ = dt.check_call(dec, truth, "D6", "decode", ids, out, pre, post, pre["seqlens"].astype(np.int64),
                                      floor_ratio=DECODE_FLOOR_RATIO)
        print(f"TRUTH lora decode step {s}: out rel-L2 {err:.3e} floor {floor:.3e}; worst stage / layer "
              + " ".join(f"{k} {v:.2e}" for k, v in worst.items()))
    dec.unload()
