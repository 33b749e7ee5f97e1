"""Chained launches of 17..64 rows at full model size against fp64: the stream-K regimes of the 32- and 64-row wgmma tiles.

At the shapes of test_gpu_wide_chain.py every wide launch takes the aligned half of gemm_tc_launch's grid rule, one segment
per CTA.  At 7B and 70B size q|k|v, gate|up and the head are stream-K (tests/wide_plan.py walk, test_wide_plan.py
test_full_cases_reach_every_regime): CTAs run 2, 3, 5 and 9 segments one after the other over the combine buffer that
overlays their pipeline rings, re-select the matrix and the RoPE mask per segment, cross from q to k and k to v, run
segments whose group-snapped range is empty or leaves one warpgroup without a group, and hand gate|up partials to a finisher
across CTAs that own other strips.  The blocks (wide_plan.FULL_BLOCKS), in the presets' own plans:
  * 7b-4.0bpw: m54 attention, the m54 MLP and the m43 MLP of every fourth layer, the 6-bit head and an 8-bit head (the
    exl2-8bpw model's 4 KB stages: 3 stages at TW 32);
  * 7b-gptq: GPTQ 4-bit g128 act-order attention and MLP, the 6-bit head;
  * 70b-2.5bpw: the 70B layer, its 32000-column head, and a 152064-column 6-bit head fed by the same MLP's chain_head.
Each block runs the decoder's chain -- q_attn_forward_2_ex -> q_mlp_forward_ex -> q_attn_forward_1_ex (NeoX RoPE at ragged
per-sequence past_lens) and q_attn_forward_2_ex -> q_mlp_forward_ex -> gemm_half_q_half_prepared -- at 64, 33, 17, 48, 24, 32
rows and 40 rows as 5 x 8 tokens.  Every stage is checked on the kernel's own previous fp16 output against fp64 (weights:
reconstruct(), checked against the oracle on column slices as test_gpu_full_shapes does; products by decoder_truth.mm64 in
column chunks), over the tensor and the worst row (test_gpu_wide_chain's bounds), against the plain forms, and per
(row, 128-column strip), where one dropped or doubled split-K partial cannot hide in a tensor-wide norm.  Also:
  * rows past M are never written: q / k / v, x and the logits are views of buffers whose rows past M (up to the tile width
    and beyond) hold sentinels, checked after every call; the 64-row step runs first, so the 33- and 17-row steps find
    stale, large token slots past M in their consumers' 64-row activation buffers;
  * determinism: the MLP runs twice per step to the same bits, one whole step twice, and a captured 7B step replays to the
    eager step's bits;
  * unit rows: zero residual and unit-vector rows of the attention output give o_proj rows of reconstruct() bit for bit.
The last test runs the shipped chained decode step on a 4-layer decoder of 7B dimensions (test_gpu_decoder_wide).
"""
import dataclasses
import time

import numpy as np
import pytest
import torch

import decoder_truth as dt
import exl2_oracle as oracle
import test_gpu_decoder_truth as tt
import test_gpu_decoder_wide as tw
import test_gpu_full_shapes as fs
import wide_plan as wp

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROWS = [64, 33, 17, 48, 24, 32, 40]     # 64 first: its token slots past M stay in the consumers' buffers for 33 and 17
PAD_ROWS = 80                           # sentinel rows after row M reach past the 64-row tile
TOL, ROW_TOL, PLAIN_TOL = 1.5e-3, 4e-3, 2e-3    # test_gpu_wide_chain.py
# per (row, 128-column strip) rel-L2 against fp64.  A strip's 128 values carry the same fp16 output rounding as a whole row, so
# its error sits near the row's: measured worst 1.05e-3 over every strip of the file (the 70B MLP output, down K = 28672), the
# rest at or below 7.9e-4 (DESIGN.md §3.7); the bound is about twice that.  One split-K partial dropped or counted twice moves
# its strip by a share of the strip's own sum (1/nc of it, nc = 2..4 contributors here), far above it.
STRIP_TOL = 2e-3
MEASURED = {}


def _note(key, v):
    MEASURED[key] = max(MEASURED.get(key, 0.0), v)


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.time()
    torch.zeros(1, device=DEV)
    torch.cuda.reset_peak_memory_stats(DEV)
    yield
    peak = torch.cuda.max_memory_allocated(DEV)
    print(f"\nWIDE-FULL wall {time.time() - t0:.0f} s, peak torch allocation {peak / 2**30:.2f} GiB")
    for k, v in sorted(MEASURED.items()):
        print(f"WIDE-FULL {k}: {v:.3e}")


def _batch(rows):
    return (5, 8) if rows == 40 else (rows, 1)


class FullBlock:
    """One layer of a wide_plan.FULL_BLOCKS block in its plans, its heads, and the chains of the decoder step."""

    def __init__(self, name):
        from exllamav2_b200 import ext as ext_c
        from exllamav2_b200.ext import none_tensor
        hid, inter, H, KVH, ap, mps, heads = wp.FULL_BLOCKS[name]
        self.name, self.hid, self.inter, self.H, self.KVH, self.hd = name, hid, inter, H, KVH, 128
        self.lin, self.W = {}, {}
        shapes = dict(q=(hid, H * 128, ap, 81), k=(hid, KVH * 128, ap, 81), v=(hid, KVH * 128, ap, 81), o=(H * 128, hid, ap, None))
        for i, mp in enumerate(mps):
            shapes.update({f"g{i}": (hid, inter, mp, 85 + i), f"u{i}": (hid, inter, mp, 85 + i), f"d{i}": (inter, hid, mp, None)})
        for j, (n, hp) in enumerate(heads):
            shapes[f"h{j}"] = (hid, n, hp, None)
        for s, (n, (K, N, p, perm)) in enumerate(shapes.items()):
            self.lin[n], self.W[n], _ = fs.load(K, N, p, 8000 + 17 * s + len(name), perm)
        self.nmlp, self.nhead = len(mps), len(heads)
        rng = np.random.default_rng(len(name))
        self.n1, self.n2, self.n3 = (torch.from_numpy((1 + 0.1 * rng.normal(size=(hid,))).astype(np.float16)).to(DEV) for _ in range(3))
        self.sin_np, self.cos_np = oracle.rope_tables(128, 512)
        self.sin, self.cos = torch.from_numpy(self.sin_np).to(DEV), torch.from_numpy(self.cos_np).to(DEV)
        h = lambda n: self.lin[n].q_handle
        self.attn = ext_c.make_q_attn(self.n1, none_tensor, True, False, 1e-5, h("q"), h("k"), h("v"), h("o"), none_tensor,
                                      none_tensor, 64, hid, H, KVH, 128, 512, True, 2, 128, none_tensor, none_tensor, none_tensor,
                                      none_tensor, False, True)
        self.ta = torch.empty((64, inter), dtype=torch.half, device=DEV)
        self.tb = torch.empty_like(self.ta)
        self.mlp = [ext_c.make_q_mlp(self.n2, none_tensor, True, 1e-5, h(f"g{i}"), h(f"u{i}"), h(f"d{i}"), none_tensor, self.ta,
                                     self.tb, none_tensor, 64, False, True, none_tensor, none_tensor, False, True)
                    for i in range(self.nmlp)]
        self.chain_mlp = [ext_c.make_chain([h(f"g{i}"), h(f"u{i}")], self.n2) for i in range(self.nmlp)]
        self.chain_attn = ext_c.make_chain([h("q"), h("k"), h("v")], self.n1)
        self.chain_head = [ext_c.make_chain([h(f"h{j}")], self.n3) for j in range(self.nhead)]

    def close(self):
        from exllamav2_b200 import ext as ext_c
        ext_c.free_q_attn(self.attn)
        for m in self.mlp:
            ext_c.free_q_mlp(m)
        for l in self.lin.values():
            l.unload()
        self.lin, self.W = {}, {}


class Padded:
    """[rows, n] views of buffers with PAD_ROWS - rows sentinel rows after them"""

    def __init__(self, seed):
        self.g = torch.Generator(device=DEV).manual_seed(seed)
        self.bufs = []

    def new(self, rows, n, init=None):
        buf = (torch.randn((PAD_ROWS, n), device=DEV, generator=self.g) * 300).half()
        if init is not None:
            buf[:rows] = init.view(rows, n)
        self.bufs.append((buf, rows, buf[rows:].clone()))
        return buf[:rows]

    def check(self, what):
        for buf, rows, want in self.bufs:
            assert torch.equal(buf[rows:].view(torch.int16), want.view(torch.int16)), f"{what}: rows past {rows} were written"


def _inputs(b, rows, seed, big_from=None):
    """x0, ao and past_lens of a step; rows from big_from on 16x larger (the stale slots the steps after the first one find)"""
    batch, q_len = _batch(rows)
    rng = np.random.default_rng(seed)
    s = np.ones((rows, 1))
    if big_from is not None:
        s[big_from:] = 16
    x0 = torch.from_numpy((s * rng.normal(0, 1, size=(rows, b.hid))).astype(np.float16)).to(DEV)
    ao = torch.from_numpy((s * rng.normal(0, 1, size=(rows, b.H * 128))).astype(np.float16)).to(DEV)
    pl = rng.integers(0, 500 - q_len, size=batch).astype(np.int32)
    pl[0] = 0
    return x0, ao, pl


def _passes(b):
    """(MLP, consumer) of each pass of a step: MLP 0 feeds q|k|v; then every head, each fed by an MLP in turn"""
    return [(0, "qkv")] + [((j + 1) % b.nmlp, j) for j in range(b.nhead)]


def _chained_step(b, rows, x0, ao, pl, pad):
    """the chained step, every output a padded view; returns {stage: tensor [rows, n]}"""
    from exllamav2_b200 import ext as ext_c
    batch, q_len = _batch(rows)
    out = {}
    for mi, cons in _passes(b):
        x = pad.new(rows, b.hid, x0)
        ext_c.q_attn_forward_2_ex(b.attn, x.view(batch, q_len, -1), ao.view(batch, q_len, -1), batch, q_len, False, b.chain_mlp[mi])
        pad.check(f"o_proj at {rows} rows")
        out[f"x1.{mi}"] = x.clone()
        ext_c.q_mlp_forward_ex(b.mlp[mi], x, True, b.chain_attn if cons == "qkv" else b.chain_head[cons])
        pad.check(f"MLP {mi} at {rows} rows")
        if f"x2.{mi}" in out:
            assert torch.equal(out[f"x2.{mi}"], x), f"MLP {mi} at {rows} rows: a second run gave different bits"
        out[f"x2.{mi}"] = x.clone()
        if cons == "qkv":
            q, k, v = pad.new(rows, b.H * 128), pad.new(rows, b.KVH * 128), pad.new(rows, b.KVH * 128)
            ext_c.q_attn_forward_1_ex(b.attn, None, batch, q_len, -1, torch.from_numpy(pl).to(DEV), q.view(batch, q_len, -1),
                                      k.view(batch, q_len, -1), v.view(batch, q_len, -1), b.sin, b.cos, True)
            pad.check(f"q|k|v at {rows} rows")
            out.update(q=q.clone(), k=k.clone(), v=v.clone())
        else:
            lg = pad.new(rows, b.W[f"h{cons}"].shape[1])
            ext_c.gemm_half_q_half_prepared(b.lin[f"h{cons}"].q_handle, lg, True, 1e-5)
            pad.check(f"head {cons} at {rows} rows")
            out[f"h{cons}"] = lg.clone()
    return out


def _plain_step(b, rows, x0, ao, pl):
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200.ext import none_tensor
    batch, q_len = _batch(rows)
    out = {}
    for mi, cons in _passes(b):
        x = x0.clone()
        ext_c.q_attn_forward_2(b.attn, x.view(batch, q_len, -1), ao.view(batch, q_len, -1), batch, q_len)
        out[f"x1.{mi}"] = x.clone()
        ext_c.q_mlp_forward_(b.mlp[mi], x)
        out[f"x2.{mi}"] = x.clone()
        if cons == "qkv":
            q = torch.empty((batch, q_len, b.H * 128), dtype=torch.half, device=DEV)
            k = torch.empty((batch, q_len, b.KVH * 128), dtype=torch.half, device=DEV)
            v = torch.empty_like(k)
            ext_c.q_attn_forward_1(b.attn, x.view(batch, q_len, -1), batch, q_len, -1, torch.from_numpy(pl).to(DEV), q, k, v,
                                   b.sin, b.cos)
            out.update(q=q.view(rows, -1), k=k.view(rows, -1), v=v.view(rows, -1))
        else:
            xn = torch.empty_like(x)
            ext_c.rms_norm(x, b.n3, xn, 1e-5)
            lg = torch.empty((rows, b.W[f"h{cons}"].shape[1]), dtype=torch.half, device=DEV)
            ext_c.gemm_half_q_half(xn, b.lin[f"h{cons}"].q_handle, lg, False)
            out[f"h{cons}"] = lg
    return out


def _norm64(x, w, eps=1e-5):
    xf = x.double()
    return xf * w.double() / torch.sqrt((xf * xf).mean(-1, keepdim=True) + eps)


def _truth(b, rows, got, x0, ao, pl):
    """fp64 of every stage on the kernel's own previous fp16 output"""
    batch, q_len = _batch(rows)
    pos = np.repeat(pl.astype(np.int64), q_len) + np.tile(np.arange(q_len), batch)
    want = {}
    for mi, cons in _passes(b):
        want[f"x1.{mi}"] = x0.double() + dt.mm64(ao, b.W["o"])
        xn = _norm64(got[f"x1.{mi}"], b.n2)
        g, u = dt.mm64(xn, b.W[f"g{mi}"]).half(), dt.mm64(xn, b.W[f"u{mi}"]).half()
        act = torch.from_numpy(oracle.silu_mul(g.cpu().numpy(), u.cpu().numpy()).astype(np.float64)).to(DEV)
        want[f"x2.{mi}"] = got[f"x1.{mi}"].double() + dt.mm64(act, b.W[f"d{mi}"])
        if cons == "qkv":
            xn1 = _norm64(got[f"x2.{mi}"], b.n1)
            for n, nh in (("q", b.H), ("k", b.KVH)):
                t = dt.mm64(xn1, b.W[n]).half().cpu().numpy().reshape(rows, nh, 128)
                want[n] = torch.from_numpy(oracle.rope_neox(t, b.sin_np, b.cos_np, pos).reshape(rows, -1).astype(np.float64)).to(DEV)
            want["v"] = dt.mm64(xn1, b.W["v"])
        else:
            want[f"h{cons}"] = dt.mm64(_norm64(got[f"x2.{mi}"], b.n3), b.W[f"h{cons}"])
    return want


def _errs(got, want):
    d = got.double() - want
    rel = (torch.linalg.norm(d) / torch.linalg.norm(want)).item()
    row = (torch.linalg.norm(d, dim=-1) / torch.linalg.norm(want, dim=-1).clamp_min(1e-30)).max().item()
    ds, ws = d.view(d.shape[0], -1, 128), want.view(want.shape[0], -1, 128)
    strip = (torch.linalg.norm(ds, dim=-1) / torch.linalg.norm(ws, dim=-1).clamp_min(1e-30)).max().item()
    return rel, row, strip


def _check_step(b, rows, seed, big_from=None):
    x0, ao, pl = _inputs(b, rows, seed, big_from)
    pad = Padded(seed)
    got = _chained_step(b, rows, x0, ao, pl, pad)
    plain = _plain_step(b, rows, x0, ao, pl)
    want = _truth(b, rows, got, x0, ao, pl)
    for nm, w in want.items():
        rel, row, strip = _errs(got[nm], w)
        e_plain = (torch.linalg.norm(got[nm].double() - plain[nm].double()) / torch.linalg.norm(plain[nm].double())).item()
        key = f"{b.name} {nm.split('.')[0]}"
        for kind, v in (("rel", rel), ("row", row), ("strip", strip), ("plain", e_plain)):
            _note(f"{key} {kind}", v)
        assert rel <= TOL, f"{key} at {rows} rows: rel-L2 {rel:.2e} vs fp64"
        assert row <= ROW_TOL, f"{key} at {rows} rows: worst row rel-L2 {row:.2e} vs fp64"
        assert strip <= STRIP_TOL, f"{key} at {rows} rows: worst (row, strip) rel-L2 {strip:.2e} vs fp64"
        assert e_plain <= PLAIN_TOL, f"{key} at {rows} rows: rel-L2 {e_plain:.2e} vs the plain form"
    return got


def _unit_rows(b, rows, seed):
    """zero residual, unit-vector rows of the attention output: o_proj through q_attn_forward_2_ex returns rows of
    reconstruct() bit for bit, whatever the split-K hand-off"""
    from exllamav2_b200 import ext as ext_c
    batch, q_len = _batch(rows)
    r = torch.from_numpy(np.random.default_rng(seed).choice(b.H * 128, rows, replace=False)).to(DEV)
    e = torch.zeros((rows, b.H * 128), dtype=torch.half, device=DEV)
    e[torch.arange(rows, device=DEV), r] = 1.0
    pad = Padded(seed)
    x = pad.new(rows, b.hid, torch.zeros((rows, b.hid), dtype=torch.half, device=DEV))
    ext_c.q_attn_forward_2_ex(b.attn, x.view(batch, q_len, -1), e.view(batch, q_len, -1), batch, q_len, False, b.chain_mlp[0])
    pad.check(f"unit rows at {rows} rows")
    assert torch.equal(x, b.W["o"][r]), f"{rows} rows: unit-vector rows of o_proj differ from the weights"


def _graph_step(b, rows):
    """one captured step (o_proj -> MLP -> q|k|v and -> MLP -> head) replays to the eager step's bits"""
    from exllamav2_b200 import ext as ext_c
    batch, q_len = _batch(rows)
    x0, ao, pl_np = _inputs(b, rows, 900)
    pl = torch.from_numpy(pl_np).to(DEV)
    s = torch.cuda.Stream(DEV)
    pad = Padded(rows)
    bufs = dict(x=pad.new(rows, b.hid), q=pad.new(rows, b.H * 128), k=pad.new(rows, b.KVH * 128), v=pad.new(rows, b.KVH * 128),
                xh=pad.new(rows, b.hid), h=pad.new(rows, b.W["h0"].shape[1]))

    def step():
        bufs["x"].copy_(x0)
        bufs["xh"].copy_(x0)
        ext_c.q_attn_forward_2_ex(b.attn, bufs["x"].view(batch, q_len, -1), ao.view(batch, q_len, -1), batch, q_len, False, b.chain_mlp[0])
        ext_c.q_mlp_forward_ex(b.mlp[0], bufs["x"], True, b.chain_attn)
        ext_c.q_attn_forward_1_ex(b.attn, None, batch, q_len, -1, pl, bufs["q"].view(batch, q_len, -1), bufs["k"].view(batch, q_len, -1),
                                  bufs["v"].view(batch, q_len, -1), b.sin, b.cos, True)
        mi = 1 % b.nmlp
        ext_c.q_attn_forward_2_ex(b.attn, bufs["xh"].view(batch, q_len, -1), ao.view(batch, q_len, -1), batch, q_len, False, b.chain_mlp[mi])
        ext_c.q_mlp_forward_ex(b.mlp[mi], bufs["xh"], True, b.chain_head[0])
        ext_c.gemm_half_q_half_prepared(b.lin["h0"].q_handle, bufs["h"], True, 1e-5)

    s.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(s):
        step()
        torch.cuda.synchronize()
        eager = {k: v.clone() for k, v in bufs.items()}
        for v in bufs.values():
            v.fill_(0)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            step()
        g.replay()
        torch.cuda.synchronize()
    pad.check(f"captured {rows}-row step")
    for k, v in bufs.items():
        assert torch.equal(v.view(torch.int16), eager[k].view(torch.int16)), f"captured {rows}-row step: {k} differs from eager"


@pytest.mark.parametrize("block", list(wp.FULL_BLOCKS))
def test_full_block_chain(block):
    """every chained entry point of a full-size block at 17..64 rows: fp64 (tensor, row, strip), plain forms, sentinel rows,
    determinism, unit rows; the 7B block also replays a captured step"""
    b = FullBlock(block)
    try:
        for rows in ROWS:
            got = _check_step(b, rows, 100 + rows, big_from=17 if rows == 64 else None)
            if rows == 33:       # one whole step twice: the same bits
                again = _chained_step(b, rows, *_inputs(b, rows, 100 + rows), Padded(0))
                for k, v in got.items():
                    assert torch.equal(v.view(torch.int16), again[k].view(torch.int16)), f"{rows} rows: a second step differs in {k}"
            _unit_rows(b, rows, rows)
        if block == "7b-4.0bpw":
            _graph_step(b, 24)
        fs._check_peak()
    finally:
        b.close()
        torch.cuda.empty_cache()


# ---- the shipped decode step at 7B dimensions -------------------------------------------------------------------------------

CASES_7B = [17, 24, 32, 64]


@pytest.mark.parametrize("B", CASES_7B)
def test_decoder_7b_wide(B, monkeypatch, request):
    """A 4-layer decoder of llama2-7b-4.0bpw dimensions and plans (layer 2 runs the m43 MLP): decode steps of 17, 24 and 32
    sequences take the chained step on the 32-row tile, 64 the 64-row tile (test_gpu_decoder_wide._forced_wide), on a ragged,
    poisoned, permuted cache; two steps against the fp64 forward (decoder_truth.check_call) and the branch (_wide_branch);
    at 17..32 the first step is followed by a graph replay against the eager step's bits, and the second step is replayed.
    The synthetic 7B stack stays in fp16 range over 4 layers (unlike the 70B one, DESIGN.md §3.7)."""
    from exllamav2_b200.model import PRESETS, ExLlamaV2Decoder
    if tt._in_child(request, True):
        return
    cfg = dataclasses.replace(PRESETS["llama2-7b-4.0bpw"](), name="llama2-7b-4.0bpw-4l", num_layers=4, max_seq_len=512)
    dec = ExLlamaV2Decoder(cfg, device=DEV, seed=fs.SEED, batch_size=B, cache_len=512, cache_bits=4)
    bt = dec.cache.block_table
    perm = torch.randperm(bt.numel(), generator=torch.Generator().manual_seed(3000 + B)).to(torch.int32)
    bt.copy_(perm.view(bt.shape).to(bt.device))
    try:
        assert dec._chains(B) == (B <= 32)
        if B > 32:
            tw._forced_wide(dec)
        truth = fs._truth(dec)
        tw._run(dec, truth, 2, monkeypatch, 700 + B, graph=B < 64)
        fs._check_peak()
    finally:
        dec.unload()
        torch.cuda.empty_cache()
