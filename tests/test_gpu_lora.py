"""LoRA adapters on the fused attention / MLP blocks (csrc/lora.cu through q_attn_set_loras / q_mlp_set_loras and the `loras`
argument of q_attn_forward_1 / _2 / q_mlp_forward_) against fp64.

Truth, per projection P with active adapters: y_P = in_P W_P (+ bias) + sum_a (in_P A_a) B_a, with in_P the RMSNorm'd block input
(q, k, v, gate, up), attn_output (o) or act(gate) . up (down); then RoPE on q and k, act(gate) . up, and the residual for o and
down.  The weights are the matrices' own reconstruction (bit-exact), A / B the fp16 values the kernel reads; everything else is
exact.  Every output within 1e-3 rel-L2.

Row counts 1 (integer GEMV), 2 / 8 (one wgmma pass), 9 / 16 (two passes), 40 (dense path); head dim 64 (GQA, NeoX) and 128
(GPT-J); SiLU and GELU with a gate / up bias; ranks 8, 16, 64, 128; adapters on q and v only and on every projection; two adapters at
once; an id registered nowhere; the Llama-2-7B shapes (large K on down, many clusters per launch).  Also: a zero B leaves
q / k / v and the O output bit-identical to the call without adapters; loras=[] on a handle with adapters is bit-identical
(and launch for launch) to a handle that never had any; set_loras replaces; a captured graph equals eager; the library's
shape checks; the reference's own call forms."""
import math

import numpy as np
import pytest
import torch

import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-3
EPS = 1e-5
ATTN = ("q_proj", "k_proj", "v_proj", "o_proj")
MLP = ("gate_proj", "up_proj", "down_proj")


def _lin(w_np, K, N):
    from exllamav2_b200.linear import ExLlamaV2Linear, load_tensor_dict
    lin = ExLlamaV2Linear(K, N, has_bias="bias" in w_np, device=DEV)
    lin.load(load_tensor_dict(w_np, DEV))
    return lin


def _f64(t):
    return t.to(torch.float64)


class Blocks:
    """One attention block and one MLP block on synthetic EXL2 matrices (q/k/v and gate/up share their row permutation, as
    converted checkpoints do)."""

    def __init__(self, hidden=512, heads=8, kv_heads=2, hd=64, inter=1408, rope_style=2, gelu=False, bias=False, seed=0):
        from exllamav2_b200 import ext
        from exllamav2_b200.ext import none_tensor
        self.hidden, self.heads, self.kvh, self.hd, self.inter = hidden, heads, kv_heads, hd, inter
        self.rope_style, self.gelu = rope_style, gelu
        # (the MLP's matrices at the existing MLP tests' scales: act(gate) * up of the default scales overflows fp16)
        mk = lambda K, N, s, b=False, sm=(0.5, 4.0): synth.make_exl2(K, N, (5, 4), (0.1, 0.9), 64, seed=seed * 10 + s, bias=b,
                                                                      scale_max_range=sm)
        wq, wk, wv, wo = mk(hidden, heads * hd, 1), mk(hidden, kv_heads * hd, 2), mk(hidden, kv_heads * hd, 3), mk(heads * hd, hidden, 4)
        wk["q_invperm"], wv["q_invperm"] = wq["q_invperm"].copy(), wq["q_invperm"].copy()
        sm = (0.02, 0.08)
        wg, wu, wd = mk(hidden, inter, 5, bias, sm), mk(hidden, inter, 6, bias, sm), mk(inter, hidden, 7, False, sm)
        wu["q_invperm"] = wg["q_invperm"].copy()
        self.lins = dict(zip(ATTN + MLP, (_lin(wq, hidden, heads * hd), _lin(wk, hidden, kv_heads * hd), _lin(wv, hidden, kv_heads * hd),
                                          _lin(wo, heads * hd, hidden), _lin(wg, hidden, inter), _lin(wu, hidden, inter),
                                          _lin(wd, inter, hidden))))
        self.W = {k: _f64(l.get_weight_tensor_dq()) for k, l in self.lins.items()}
        self.bias = {k: torch.from_numpy(w["bias"].astype(np.float64)).to(DEV) for k, w in (("gate_proj", wg), ("up_proj", wu)) if "bias" in w}
        rng = np.random.default_rng(seed + 5)
        self.n1 = torch.from_numpy((1 + 0.1 * rng.normal(size=(hidden,))).astype(np.float16)).to(DEV)
        self.n2 = torch.from_numpy((1 + 0.1 * rng.normal(size=(hidden,))).astype(np.float16)).to(DEV)
        ang = np.arange(256)[:, None] * (1.0 / 10000 ** (np.arange(0, hd, 2) / hd))[None, :]
        ang = np.concatenate([ang, ang], -1) if rope_style == 2 else np.repeat(ang, 2, axis=-1)
        self.sin = torch.from_numpy(np.sin(ang).astype(np.float16)).to(DEV)
        self.cos = torch.from_numpy(np.cos(ang).astype(np.float16)).to(DEV)
        self.ta = torch.empty((64, inter), dtype=torch.half, device=DEV)
        self.tb = torch.empty_like(self.ta)
        L = self.lins
        self.attn = ext.make_q_attn(self.n1, none_tensor, True, False, EPS, L["q_proj"].q_handle, L["k_proj"].q_handle,
                                    L["v_proj"].q_handle, L["o_proj"].q_handle, none_tensor, none_tensor, 64, hidden, heads, kv_heads,
                                    hd, 256, True, rope_style, hd, none_tensor, none_tensor, none_tensor, none_tensor, False, True)
        self.mlp = ext.make_q_mlp(self.n2, none_tensor, True, EPS, L["gate_proj"].q_handle, L["up_proj"].q_handle,
                                  L["down_proj"].q_handle, none_tensor, self.ta, self.tb, none_tensor, 64, gelu, True, none_tensor,
                                  none_tensor, False, True)
        self.adapters = {}

    def shape(self, proj):
        return self.lins[proj].in_features, self.lins[proj].out_features

    def adapter(self, rank, targets, seed, zero_b=False):
        """A [in, rank], B [rank, out] fp16 per target, sized so the delta is ~20 % of the projection's output: in W has
        sqrt(K) x std(W) times the input's scale, (in A) B with A ~ N(0, 1/K) has sqrt(rank) x std(B) times it."""
        g = torch.Generator(device=DEV).manual_seed(seed)
        ad = {}
        for t in targets:
            K, N = self.shape(t)
            a = (torch.randn((K, rank), device=DEV, generator=g) / math.sqrt(K)).half()
            b = (torch.randn((rank, N), device=DEV, generator=g) * (0.2 * math.sqrt(K) * self.W[t].std().item() / math.sqrt(rank))).half()
            ad[t] = (a, b.zero_() if zero_b else b)
        return ad

    def set(self, adapters: dict):
        """adapters: id -> {projection: (A, B)}; registers the whole set on both handles."""
        from exllamav2_b200 import ext
        self.adapters = adapters
        d = {t: ({k: ad[t][0] for k, ad in adapters.items() if t in ad}, {k: ad[t][1] for k, ad in adapters.items() if t in ad})
             for t in ATTN + MLP}
        r1 = ext.q_attn_set_loras(self.attn, *d["q_proj"], *d["k_proj"], *d["v_proj"], *d["o_proj"])
        r2 = ext.q_mlp_set_loras(self.mlp, *d["gate_proj"], *d["up_proj"], *d["down_proj"])
        return r1, r2

    # ---- the blocks ----
    def attn1(self, x, B, T, past, loras, past_lens=None):
        from exllamav2_b200 import ext
        from exllamav2_b200.ext import none_tensor
        q = torch.empty((B, T, self.heads * self.hd), dtype=torch.half, device=DEV)
        k = torch.empty((B, T, self.kvh * self.hd), dtype=torch.half, device=DEV)
        v = torch.empty_like(k)
        ext.q_attn_forward_1(self.attn, x, B, T, past, none_tensor if past_lens is None else past_lens, q, k, v, self.sin, self.cos,
                             loras)
        return q, k, v

    def attn2(self, x, ao, B, T, loras):
        from exllamav2_b200 import ext
        x = x.clone()
        ext.q_attn_forward_2(self.attn, x, ao, B, T, loras)
        return x

    def mlp_fwd(self, x, loras):
        from exllamav2_b200 import ext
        x = x.clone()
        rows = x.numel() // x.shape[-1]
        if rows <= self.ta.shape[0]:
            ext.q_mlp_forward_(self.mlp, x, loras)
        else:
            ta = torch.empty((rows, self.inter), dtype=torch.half, device=DEV)
            ext.q_mlp_forward_rows(self.mlp, x, ta, torch.empty_like(ta), loras)
        return x

    # ---- fp64 truth ----
    def delta(self, inp, proj, loras):
        d = 0.0
        for key in loras:
            ad = self.adapters.get(key, {})
            if proj in ad:
                a, b = ad[proj]
                d = d + (inp @ _f64(a)) @ _f64(b)
        return d

    def norm(self, x, w):
        x = _f64(x)
        return x / (x * x).mean(-1, keepdim=True).add(EPS).sqrt() * _f64(w)

    def rope(self, t, heads, pos):
        hd = self.hd
        t = t.view(-1, heads, hd)
        c, s = _f64(self.cos)[pos][:, None, :], _f64(self.sin)[pos][:, None, :]
        if self.rope_style == 2:
            h = hd // 2
            l, r = t[..., :h], t[..., h:]
            return torch.cat([l * c[..., :h] - r * s[..., :h], r * c[..., :h] + l * s[..., :h]], -1).view(t.shape[0], -1)
        x0, x1 = t[..., 0::2], t[..., 1::2]
        out = torch.empty_like(t)
        out[..., 0::2] = x0 * c[..., 0::2] - x1 * s[..., 0::2]
        out[..., 1::2] = x1 * c[..., 1::2] + x0 * s[..., 1::2]
        return out.view(t.shape[0], -1)

    def truth_attn1(self, x, pos, loras):
        xn = self.norm(x.view(-1, self.hidden), self.n1)
        y = {p: xn @ self.W[p] + self.delta(xn, p, loras) for p in ATTN[:3]}
        return self.rope(y["q_proj"], self.heads, pos), self.rope(y["k_proj"], self.kvh, pos), y["v_proj"]

    def truth_attn2(self, x, ao, loras):
        a = _f64(ao).view(-1, self.heads * self.hd)
        return _f64(x).view(-1, self.hidden) + a @ self.W["o_proj"] + self.delta(a, "o_proj", loras)

    def act(self, g):
        if self.gelu:
            return 0.5 * g * (1 + torch.tanh(0.7978845608028654 * (g + 0.044715 * g ** 3)))
        return g / (1 + torch.exp(-g))

    def truth_mlp(self, x, loras):
        x = _f64(x).view(-1, self.hidden)
        xn = self.norm(x, self.n2)
        g = xn @ self.W["gate_proj"] + self.bias.get("gate_proj", 0.0) + self.delta(xn, "gate_proj", loras)
        u = xn @ self.W["up_proj"] + self.bias.get("up_proj", 0.0) + self.delta(xn, "up_proj", loras)
        a = self.act(g) * u
        return x + a @ self.W["down_proj"] + self.delta(a, "down_proj", loras)

    def free(self):
        from exllamav2_b200 import ext
        ext.free_q_attn(self.attn)
        ext.free_q_mlp(self.mlp)
        for l in self.lins.values():
            l.unload()


def _rel(got, want) -> float:
    g = _f64(got).reshape(want.shape)
    return ((g - want).norm() / want.norm()).item()


_BLOCKS = {}


def _blocks(cfg):
    if cfg not in _BLOCKS:
        if cfg == "hd64-gqa-neox":
            _BLOCKS[cfg] = Blocks(512, 8, 2, 64, 1408, 2, gelu=False, bias=False, seed=1)
        elif cfg == "hd128-gptj-gelu-bias":
            _BLOCKS[cfg] = Blocks(1024, 8, 8, 128, 2816, 1, gelu=True, bias=True, seed=2)
        elif cfg == "llama7b":
            _BLOCKS[cfg] = Blocks(4096, 32, 32, 128, 11008, 2, gelu=False, bias=False, seed=3)
        else:
            raise KeyError(cfg)
    return _BLOCKS[cfg]


# adapter sets: name -> [(id, rank, targets)]; 999 is an id registered nowhere
SETS = {
    "qv16": [(11, 16, ("q_proj", "v_proj"))],
    "all8+qv64": [(21, 8, ATTN + MLP), (22, 64, ("q_proj", "v_proj", "gate_proj", "down_proj"))],
    "gu16": [(31, 16, ("gate_proj", "up_proj"))],
    "down64": [(41, 64, ("down_proj",))],
    "qkv128": [(51, 128, ("q_proj", "k_proj", "v_proj"))],      # 384 stacked columns: a one-adapter set above 256
}


def _activate(blk, name, zero_b=False):
    ads = {key: blk.adapter(r, t, seed=key, zero_b=zero_b) for key, r, t in SETS[name]}
    blk.set(ads)
    return [key for key, _, _ in SETS[name]] + [999]


ROWS = [1, 2, 8, 9, 16, 40]


def _split(rows):
    """rows as (batch, q_len): several sequences where the row count allows (per-sequence positions)"""
    return (2, rows // 2) if rows % 2 == 0 and rows > 1 else (1, rows)


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("cfg", ["hd64-gqa-neox", "hd128-gptj-gelu-bias"])
@pytest.mark.parametrize("adapters", ["qv16", "all8+qv64", "qkv128"])
def test_attn_block_vs_fp64(rows, cfg, adapters):
    blk = _blocks(cfg)
    loras = _activate(blk, adapters)
    B, T = _split(rows)
    rng = np.random.default_rng(rows)
    x = torch.from_numpy(rng.normal(0, 1, size=(B, T, blk.hidden)).astype(np.float16)).to(DEV)
    past_lens = torch.tensor([5 + 17 * b for b in range(B)], dtype=torch.int32, device=DEV)
    q, k, v = blk.attn1(x, B, T, -1, loras, past_lens)
    pos = torch.as_tensor(np.concatenate([5 + 17 * b + np.arange(T) for b in range(B)]), device=DEV)
    for got, want, nm in zip((q, k, v), blk.truth_attn1(x, pos, loras), "qkv"):
        err = _rel(got, want)
        assert err <= TOL, f"{nm}: rel-L2 {err:.2e}"
    ao = torch.from_numpy(rng.normal(0, 1, size=(B, T, blk.heads * blk.hd)).astype(np.float16)).to(DEV)
    x2 = blk.attn2(x, ao, B, T, loras)
    err = _rel(x2, blk.truth_attn2(x, ao, loras))
    assert err <= TOL, f"o: rel-L2 {err:.2e}"


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("cfg", ["hd64-gqa-neox", "hd128-gptj-gelu-bias"])
@pytest.mark.parametrize("adapters", ["all8+qv64", "gu16", "down64"])
def test_mlp_block_vs_fp64(rows, cfg, adapters):
    blk = _blocks(cfg)
    loras = _activate(blk, adapters)
    rng = np.random.default_rng(rows + 100)
    x = torch.from_numpy(rng.normal(0, 1, size=(rows, blk.hidden)).astype(np.float16)).to(DEV)
    got = blk.mlp_fwd(x, loras)
    want = blk.truth_mlp(x, loras)
    err = _rel(got, want)
    assert err <= TOL, f"rel-L2 {err:.2e}"
    # the adapters are visible: the same call without them is well off the adapted truth
    assert _rel(blk.mlp_fwd(x, []), want) > 3 * TOL


@pytest.mark.parametrize("rows", [1, 4, 9, 40])
def test_zero_b_bit_identical(rows):
    """B = 0 on every projection: q / k / v (RoPE'd by the LoRA launch) and the O output carry the LoRA-off bits."""
    blk = _blocks("hd64-gqa-neox")
    loras = _activate(blk, "all8+qv64", zero_b=True)
    rng = np.random.default_rng(rows + 7)
    x = torch.from_numpy(rng.normal(0, 1, size=(1, rows, blk.hidden)).astype(np.float16)).to(DEV)
    ao = torch.from_numpy(rng.normal(0, 1, size=(1, rows, blk.heads * blk.hd)).astype(np.float16)).to(DEV)
    for a, b in zip(blk.attn1(x, 1, rows, 3, loras), blk.attn1(x, 1, rows, 3, [])):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    assert torch.equal(blk.attn2(x, ao, 1, rows, loras).view(torch.int16), blk.attn2(x, ao, 1, rows, []).view(torch.int16))


@pytest.mark.parametrize("rows", [1, 8, 40])
def test_no_active_adapter_is_the_plain_path(rows):
    """loras=[] (and a list of ids registered nowhere) on a handle with adapters set: the bits and the launches of a handle that
    never had adapters."""
    from exllamav2_b200 import ext
    plain = Blocks(512, 8, 2, 64, 1408, 2, seed=1)
    blk = _blocks("hd64-gqa-neox")
    _activate(blk, "all8+qv64")
    rng = np.random.default_rng(rows + 9)
    x = torch.from_numpy(rng.normal(0, 1, size=(1, rows, blk.hidden)).astype(np.float16)).to(DEV)
    ao = torch.from_numpy(rng.normal(0, 1, size=(1, rows, blk.heads * blk.hd)).astype(np.float16)).to(DEV)

    def run(b, loras):
        torch.cuda.synchronize()
        n0 = ext.launch_count()
        out = (*b.attn1(x, 1, rows, 3, loras), b.attn2(x, ao, 1, rows, loras), b.mlp_fwd(x.view(rows, -1), loras))
        torch.cuda.synchronize()
        return out, ext.launch_count() - n0

    want, n_want = run(plain, [])
    for loras in ([], [999, 12345]):
        got, n_got = run(blk, loras)
        assert n_got == n_want
        for g, w in zip(got, want):
            assert torch.equal(g.view(torch.int16), w.view(torch.int16))
    plain.free()


def test_set_loras_replaces():
    blk = _blocks("hd64-gqa-neox")
    rng = np.random.default_rng(3)
    x = torch.from_numpy(rng.normal(0, 1, size=(4, blk.hidden)).astype(np.float16)).to(DEV)
    off = blk.mlp_fwd(x, [])
    first = {1: blk.adapter(16, ATTN + MLP, seed=1)}
    second = {2: blk.adapter(16, ATTN + MLP, seed=2)}
    assert blk.set(first) == (16, 16)
    y1 = blk.mlp_fwd(x, [1, 2])
    assert blk.set(second) == (16, 16)
    y2 = blk.mlp_fwd(x, [1, 2])                 # adapter 1 is gone: only 2 applies
    assert _rel(y2, blk.truth_mlp(x, [2])) <= TOL
    assert not torch.equal(y1, y2)
    assert blk.set({}) == (0, 0)
    assert torch.equal(blk.mlp_fwd(x, [1, 2]).view(torch.int16), off.view(torch.int16))


@pytest.mark.parametrize("rows", [1, 8])
def test_graph_equals_eager(rows):
    blk = _blocks("hd64-gqa-neox")
    loras = _activate(blk, "all8+qv64")
    rng = np.random.default_rng(rows + 11)
    x = torch.from_numpy(rng.normal(0, 1, size=(1, rows, blk.hidden)).astype(np.float16)).to(DEV)
    ao = torch.from_numpy(rng.normal(0, 1, size=(1, rows, blk.heads * blk.hd)).astype(np.float16)).to(DEV)

    def step():
        q, k, v = blk.attn1(x, 1, rows, 3, loras)
        return q, k, v, blk.attn2(x, ao, 1, rows, loras), blk.mlp_fwd(x.view(rows, -1), loras)

    eager = [t.clone() for t in step()]
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        step()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            outs = step()
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, outs):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_library_shape_checks():
    """What only the library can check: A / B against the handle's matrices."""
    blk = _blocks("hd64-gqa-neox")
    K, N = blk.shape("q_proj")
    a = torch.zeros((K + 8, 8), dtype=torch.half, device=DEV)
    b = torch.zeros((8, N), dtype=torch.half, device=DEV)
    from exllamav2_b200 import ext
    with pytest.raises(RuntimeError, match="the matrix is"):
        ext.q_attn_set_loras(blk.attn, {1: a}, {1: b}, {}, {}, {}, {}, {}, {})
    a = torch.zeros((K, 8), dtype=torch.half, device=DEV)
    b = torch.zeros((8, N + 2), dtype=torch.half, device=DEV)
    with pytest.raises(RuntimeError, match="the matrix is"):
        ext.q_attn_set_loras(blk.attn, {1: a}, {1: b}, {}, {}, {}, {}, {}, {})
    # a set whose ranks would pass the stage bound if all were active: 5 x 112 on q|k|v
    big = {i: blk.adapter(112, ("q_proj",), seed=i) for i in range(5)}
    with pytest.raises(RuntimeError, match="512"):
        blk.set(big)
    with pytest.raises(RuntimeError, match="incorrect datatype"):
        ext.q_attn_set_loras(blk.attn, {1: a.float()}, {1: b.float()}, {}, {}, {}, {}, {}, {})


def test_reference_call_forms():
    """attn.py:1545-1564 / mlp.py:520-536 (set_loras with dicts keyed by id(lora), temp_lora_size = max rank x max batch x max
    input length) and attn.py:528-548 / mlp.py:345-356 (forwards with [id(x) for x in loras] and a temp of that size)."""
    from exllamav2_b200 import ext as ext_c
    blk = _blocks("hd64-gqa-neox")

    class Lora:          # stands for ExLlamaV2Lora: the dict keys are id(lora)
        pass

    lora = Lora()
    ad = blk.adapter(16, ATTN + MLP, seed=5)
    blk.adapters = {id(lora): ad}
    g = lambda t, i: {id(lora): ad[t][i]}
    temp_lora_size = ext_c.q_attn_set_loras(blk.attn, g("q_proj", 0), g("q_proj", 1), g("k_proj", 0), g("k_proj", 1),
                                            g("v_proj", 0), g("v_proj", 1), g("o_proj", 0), g("o_proj", 1))
    temp_lora_size *= 1 * 16
    mlp_size = ext_c.q_mlp_set_loras(blk.mlp, g("gate_proj", 0), g("gate_proj", 1), g("up_proj", 0), g("up_proj", 1),
                                     g("down_proj", 0), g("down_proj", 1)) * 1 * 16
    assert temp_lora_size == mlp_size == 256
    loras = [lora]
    pass_loras = [id(x) for x in loras]
    pass_lora_temp = torch.empty((temp_lora_size,), dtype=torch.half, device=DEV)
    batch_size, q_len = 1, 5
    rng = np.random.default_rng(21)
    hidden_states = torch.from_numpy(rng.normal(0, 1, size=(batch_size, q_len, blk.hidden)).astype(np.float16)).to(DEV)
    cache_seqlens_rope = torch.tensor([12], dtype=torch.int32, device=DEV)
    q = torch.empty((batch_size, q_len, blk.heads * blk.hd), dtype=torch.half, device=DEV)
    k = torch.empty((batch_size, q_len, blk.kvh * blk.hd), dtype=torch.half, device=DEV)
    v = torch.empty_like(k)
    ext_c.q_attn_forward_1(blk.attn, hidden_states, batch_size, q_len, 0, cache_seqlens_rope, q, k, v, blk.sin, blk.cos,
                           pass_loras, pass_lora_temp)
    pos = torch.arange(12, 12 + q_len, device=DEV)
    for got, want in zip((q, k, v), blk.truth_attn1(hidden_states, pos, pass_loras)):
        assert _rel(got, want) <= TOL
    attn_output = torch.from_numpy(rng.normal(0, 1, size=(batch_size, q_len, blk.heads * blk.hd)).astype(np.float16)).to(DEV)
    x = hidden_states.clone()
    ext_c.q_attn_forward_2(blk.attn, x, attn_output, batch_size, q_len, pass_loras, pass_lora_temp)
    assert _rel(x, blk.truth_attn2(hidden_states, attn_output, pass_loras)) <= TOL
    x = hidden_states.clone()
    ext_c.q_mlp_forward_(blk.mlp, x, pass_loras, pass_lora_temp)
    assert _rel(x, blk.truth_mlp(hidden_states, pass_loras)) <= TOL


@pytest.mark.parametrize("rows", [1, 8, 40])
def test_llama7b_shapes_vs_fp64(rows):
    """Llama-2-7B shapes (hidden 4096, 32 heads of 128, intermediate 11008): K = 11008 on down stages 1376 rows of input per CTA
    (44 KB at 8 rows), and the q|k|v / gate|up launches split their columns over 12 / 16 clusters."""
    blk = _blocks("llama7b")
    loras = _activate(blk, "all8+qv64")
    rng = np.random.default_rng(rows + 200)
    x = torch.from_numpy(rng.normal(0, 1, size=(1, rows, blk.hidden)).astype(np.float16)).to(DEV)
    q, k, v = blk.attn1(x, 1, rows, 11, loras)
    pos = torch.arange(11, 11 + rows, device=DEV)
    for got, want, nm in zip((q, k, v), blk.truth_attn1(x, pos, loras), "qkv"):
        err = _rel(got, want)
        assert err <= TOL, f"{nm}: rel-L2 {err:.2e}"
    ao = torch.from_numpy(rng.normal(0, 1, size=(1, rows, blk.heads * blk.hd)).astype(np.float16)).to(DEV)
    err = _rel(blk.attn2(x, ao, 1, rows, loras), blk.truth_attn2(x, ao, loras))
    assert err <= TOL, f"o: rel-L2 {err:.2e}"
    xm = x.view(rows, -1)
    want = blk.truth_mlp(xm, loras)
    err = _rel(blk.mlp_fwd(xm, loras), want)
    assert err <= TOL, f"mlp: rel-L2 {err:.2e}"
    assert _rel(blk.mlp_fwd(xm, []), want) > 3 * TOL
