"""fp64 restatement of one ExLlamaV2Decoder call (exllamav2_b200/model.py), teacher-forced on the K/V the decoder stored.

Plain math throughout, not the fp16-rounded oracle ops: embedding row -> per layer [RMSNorm -> q/k/v = xn W -> NeoX RoPE at the
token's absolute position -> causal GQA attention with scale 1/sqrt(hd) -> o_proj + residual -> RMSNorm -> SiLU(gate) * up ->
down + residual] -> final RMSNorm -> LM head.

Positions before the call's first token come from the caller (the decoder's own cache bytes, dequantised): the truth of a call
is then a continuous function of its inputs, so a kernel that is a little off cannot hide behind a free-running sequence that
drifted across a quantisation step.  The call's own tokens enter attention unquantised, as they do in the fused kernel.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

F64 = np.float64


@dataclass
class TruthLayer:
    input_norm: np.ndarray       # [hidden]
    post_norm: np.ndarray        # [hidden]
    wq: np.ndarray               # [hidden, H * hd]      (x @ W, as the decoder's matrices are stored)
    wk: np.ndarray               # [hidden, KVH * hd]
    wv: np.ndarray
    wo: np.ndarray               # [H * hd, hidden]
    wg: np.ndarray               # [hidden, intermediate]
    wu: np.ndarray
    wd: np.ndarray               # [intermediate, hidden]


@dataclass
class CallTruth:
    hidden: np.ndarray           # [T, hidden]: residual stream after the last layer (what prefill returns)
    logits: np.ndarray           # [T, vocab]
    k: list                      # per layer [T, KVH, hd]: the call's keys after RoPE (what the cache stores)
    v: list                      # per layer [T, KVH, hd]


def rms_norm(x: np.ndarray, w: np.ndarray, eps: float) -> np.ndarray:
    x = np.asarray(x, dtype=F64)
    return x / np.sqrt((x * x).mean(-1, keepdims=True) + eps) * np.asarray(w, dtype=F64)


def rope_neox(x: np.ndarray, sin: np.ndarray, cos: np.ndarray, pos: np.ndarray) -> np.ndarray:
    """x [T, heads, hd], pos [T]: rotate the pair (i, i + hd/2) by the table's angle for frequency i at pos."""
    x = np.asarray(x, dtype=F64)
    h = x.shape[-1] // 2
    c = np.asarray(cos, dtype=F64)[pos, :h][:, None, :]
    s = np.asarray(sin, dtype=F64)[pos, :h][:, None, :]
    l, r = x[..., :h], x[..., h:]
    return np.concatenate([l * c - r * s, r * c + l * s], axis=-1)


def silu(x: np.ndarray) -> np.ndarray:
    return x / (1.0 + np.exp(-x))


def attention(q: np.ndarray, k: np.ndarray, v: np.ndarray, n_past: int) -> np.ndarray:
    """q [T, H, hd] at positions n_past .. n_past + T - 1; k / v [n_past + T, KVH, hd].  Query i sees keys [0, n_past + i]."""
    T, H, hd = q.shape
    KVH = k.shape[1]
    kk = np.repeat(k, H // KVH, axis=1)              # head h reads kv head h // (H / KVH)
    vv = np.repeat(v, H // KVH, axis=1)
    s = np.einsum("thd,nhd->htn", q, kk) / np.sqrt(hd)
    mask = np.arange(k.shape[0])[None, :] > (n_past + np.arange(T))[:, None]
    s = np.where(mask[None], -np.inf, s)
    s = s - s.max(-1, keepdims=True)
    p = np.exp(s)
    p /= p.sum(-1, keepdims=True)
    return np.einsum("htn,nhd->thd", p, vv)


class TruthModel:
    def __init__(self, layers: list, final_norm, head, embed, sin, cos, num_heads: int, num_kv_heads: int, head_dim: int,
                 eps: float):
        self.layers = layers
        self.final_norm = np.asarray(final_norm, dtype=F64)
        self.head = np.asarray(head, dtype=F64)
        self.embed = np.asarray(embed, dtype=F64)
        self.sin, self.cos = np.asarray(sin, dtype=F64), np.asarray(cos, dtype=F64)
        self.H, self.KVH, self.hd, self.eps = num_heads, num_kv_heads, head_dim, eps

    def forward(self, ids, start: int, past_k: list, past_v: list, fp16: bool = False) -> CallTruth:
        """One sequence's call over tokens `ids` at positions [start, start + T).  past_k / past_v: per layer [start, KVH, hd]
        (keys already rotated, as the cache holds them).

        fp16=True rounds every intermediate a kernel stores (normed input, projections, rotated q / k, attention output, o_proj,
        residual stream, gate / up, activation, down) to fp16 and computes everything else exactly: an ideal fp16-storage
        implementation.  Its distance from the exact forward is the fp16 floor of this input -- how far rounding alone moves
        it, which is large where the residual stream cancels."""
        ids = np.asarray(ids).reshape(-1)
        T = ids.shape[0]
        H, KVH, hd = self.H, self.KVH, self.hd
        r = _round16 if fp16 else (lambda a: a)
        pos = start + np.arange(T)
        x = self.embed[ids].copy()
        ks, vs = [], []
        for li, L in enumerate(self.layers):
            assert past_k[li].shape[0] == start and past_v[li].shape[0] == start
            xn = r(rms_norm(x, L.input_norm, self.eps))
            q = r(rope_neox(r(xn @ L.wq).reshape(T, H, hd), self.sin, self.cos, pos))
            k = r(rope_neox(r(xn @ L.wk).reshape(T, KVH, hd), self.sin, self.cos, pos))
            v = r((xn @ L.wv).reshape(T, KVH, hd))
            ks.append(k)
            vs.append(v)
            kc = np.concatenate([np.asarray(past_k[li], dtype=F64), k])
            vc = np.concatenate([np.asarray(past_v[li], dtype=F64), v])
            o = r(attention(q, kc, vc, start).reshape(T, H * hd))
            x = r(x + r(o @ L.wo))
            xn = r(rms_norm(x, L.post_norm, self.eps))
            a = r(silu(r(xn @ L.wg)) * r(xn @ L.wu))
            x = r(x + r(a @ L.wd))
        logits = rms_norm(x, self.final_norm, self.eps) @ self.head
        return CallTruth(hidden=x, logits=logits, k=ks, v=vs)


def _round16(a: np.ndarray) -> np.ndarray:
    return np.asarray(a).astype(np.float16).astype(F64)


# ---- the same forward in torch fp64, for models whose fp64 weights do not fit anywhere --------------------------------------
# Weights stay in whatever dtype the caller holds them (the decoder's fp16 reconstruct() on the GPU); every product converts one
# column chunk of at most CHUNK_BYTES of fp64 at a time, so a 70B-shaped layer never exists in fp64 as a whole.

CHUNK_BYTES = 512 << 20


def mm64(a, w, chunk_bytes: int = CHUNK_BYTES):
    """a [T, K] @ w [K, N] in fp64, w converted to fp64 one column chunk at a time."""
    import torch
    a = a.to(torch.float64)
    K, N = w.shape
    cols = max(1, chunk_bytes // (8 * K))
    out = torch.empty((a.shape[0], N), dtype=torch.float64, device=a.device)
    for j0 in range(0, N, cols):
        out[:, j0:j0 + cols] = a @ w[:, j0:j0 + cols].to(torch.float64)
    return out


class TorchTruthModel:
    """TruthModel.forward restated in torch fp64 on `device` (tests/test_decoder_truth_model.py pins the two together).  layers:
    TruthLayer-like objects whose matrices are torch tensors [K, N] of any float dtype; the result is a numpy CallTruth."""

    def __init__(self, layers: list, final_norm, head, embed, sin, cos, num_heads: int, num_kv_heads: int, head_dim: int,
                 eps: float, device, chunk_bytes: int = CHUNK_BYTES):
        import torch
        f = lambda t: torch.as_tensor(t).to(device=device, dtype=torch.float64)
        self.layers = layers
        self.norms = [(f(L.input_norm), f(L.post_norm)) for L in layers]
        self.final_norm, self.head, self.embed = f(final_norm), head, torch.as_tensor(embed).to(device)     # rows converted when read
        self.sin, self.cos = f(sin), f(cos)
        self.H, self.KVH, self.hd, self.eps, self.device = num_heads, num_kv_heads, head_dim, eps, device
        self.chunk = chunk_bytes

    def _norm(self, x, w):
        return x / (x * x).mean(-1, keepdim=True).add(self.eps).sqrt() * w

    def _rope(self, x, pos):
        import torch
        h = x.shape[-1] // 2
        c, s = self.cos[pos, :h][:, None, :], self.sin[pos, :h][:, None, :]
        l, r = x[..., :h], x[..., h:]
        return torch.cat([l * c - r * s, r * c + l * s], dim=-1)

    def forward(self, ids, start: int, past_k: list, past_v: list, fp16: bool = False) -> CallTruth:
        import torch
        ids = np.asarray(ids).reshape(-1)
        T = ids.shape[0]
        H, KVH, hd = self.H, self.KVH, self.hd
        r = (lambda a: a.half().double()) if fp16 else (lambda a: a)
        pos = torch.as_tensor(start + np.arange(T), device=self.device)
        x = self.embed[torch.as_tensor(ids, device=self.device)].to(torch.float64)
        ks, vs = [], []
        mask = torch.arange(start + T, device=self.device)[None, :] > pos[:, None]
        for li, L in enumerate(self.layers):
            n1, n2 = self.norms[li]
            assert past_k[li].shape[0] == start and past_v[li].shape[0] == start
            xn = r(self._norm(x, n1))
            q = r(self._rope(r(mm64(xn, L.wq, self.chunk)).view(T, H, hd), pos))
            k = r(self._rope(r(mm64(xn, L.wk, self.chunk)).view(T, KVH, hd), pos))
            v = r(mm64(xn, L.wv, self.chunk).view(T, KVH, hd))
            ks.append(k.cpu().numpy())
            vs.append(v.cpu().numpy())
            kc = torch.cat([torch.as_tensor(np.asarray(past_k[li], dtype=F64), device=self.device), k])
            vc = torch.cat([torch.as_tensor(np.asarray(past_v[li], dtype=F64), device=self.device), v])
            kk = kc.repeat_interleave(H // KVH, dim=1)          # head h reads kv head h // (H / KVH)
            vv = vc.repeat_interleave(H // KVH, dim=1)
            s = torch.einsum("thd,nhd->htn", q, kk) / math.sqrt(hd)
            s = s.masked_fill(mask[None], -math.inf)
            p = torch.softmax(s, dim=-1)
            o = r(torch.einsum("htn,nhd->thd", p, vv).reshape(T, H * hd))
            x = r(x + r(mm64(o, L.wo, self.chunk)))
            xn = r(self._norm(x, n2))
            g, u = r(mm64(xn, L.wg, self.chunk)), r(mm64(xn, L.wu, self.chunk))
            a = r(g / (1.0 + torch.exp(-g)) * u)
            x = r(x + r(mm64(a, L.wd, self.chunk)))
        logits = mm64(self._norm(x, self.final_norm), self.head, self.chunk)
        return CallTruth(hidden=x.cpu().numpy(), logits=logits.cpu().numpy(), k=ks, v=vs)


# ---- which host branch a decoder call ran (shared by the GPU decoder tests) ------------------------------------------------------------------------------------------------

SPIED = ["q_attn_forward_1", "q_attn_forward_1_ex", "paged_attn_decode_q4", "q_mlp_forward_", "q_mlp_forward_ex",
         "q_mlp_forward_rows", "gemv_norm", "gemm_half_q_half_prepared", "gemm_half_q_half", "rms_norm", "q_to_fp16_kv",
         "fp16_to_q_kv"]


class Spy:
    """Records the extension entry points the decoder calls (name, args, kwargs) without changing what they do."""

    def __init__(self, monkeypatch):
        from exllamav2_b200 import ext, model
        self.calls = []
        for name in SPIED:
            monkeypatch.setattr(ext, name, self._wrap(name, getattr(ext, name)))
        monkeypatch.setattr(model, "_sdpa_prefill", self._wrap("_sdpa_prefill", model._sdpa_prefill))
        monkeypatch.setattr(model._lib, "exl2b_paged_attn_decode", self._wrap("exl2b_paged_attn_decode", model._lib.exl2b_paged_attn_decode))

    def _wrap(self, name, fn):
        def w(*a, **kw):
            self.calls.append((name, a, kw))
            return fn(*a, **kw)
        return w

    def take(self):
        c, self.calls = self.calls, []
        return c


def named(calls, name):
    return [(a, kw) for n, a, kw in calls if n == name]


def names_of(calls):
    return {n for n, _, _ in calls}


def check_branch(sched, kind, calls, dec, L):
    """Assert the host branch a call took, from the entry points it reached."""
    from exllamav2_b200 import ext, model
    B = dec.batch_size
    # above one row the chained schedule runs every matrix on the wgmma kernel: a model with a matrix it cannot stage takes the
    # fused, un-chained branch there instead (D5 as D3 / D6, P1 through q_attn_forward_1)
    staged = all(ext.qmatrix_tc_supported(l.q_handle) for l in dec.linears)
    if not staged and sched == "D5":
        sched = "D6"
    names = names_of(calls)
    attn1 = named(calls, "q_attn_forward_1")
    attn1_ex = named(calls, "q_attn_forward_1_ex")
    fused = named(calls, "paged_attn_decode_q4")
    ref_attn = named(calls, "exl2b_paged_attn_decode")
    rows1 = sorted({a[2] * a[3] for a, _ in attn1})          # batch_size * q_len of q_attn_forward_1
    if sched == "L" and kind == "decode":                    # the long case decodes in the benchmarked step
        sched = "D1"
    if kind == "decode":
        head = {"gemv_norm", "gemm_half_q_half_prepared", "gemm_half_q_half"} & names
        if sched == "D1":
            assert dec.row_gemv and dec.chained and dec.fused_attn and B == 1
            assert len(attn1_ex) == L and all(a[9] is None for a, _ in attn1_ex), "RoPE must be left to the attention kernel"
            assert len(fused) == L and all(kw.get("rope") is not None for _, kw in fused)
            assert head == {"gemv_norm"} and named(calls, "gemv_norm")[0][1].get("prepared") is True
        elif sched in ("D2", "D5"):
            assert dec.chained and dec.fused_attn and B <= 8 and (B > 1 or not dec.row_gemv)
            assert len(attn1_ex) == L and all(a[9] is not None and a[2] == B for a, _ in attn1_ex)
            assert len(fused) == L and all(kw.get("rope") is None for _, kw in fused)
            assert head == {"gemm_half_q_half_prepared"}
        elif sched in ("D3", "D6"):
            assert dec.fused_attn and not (dec.chained and B <= 8 and staged)
            assert not attn1_ex and rows1 == [B] and len(fused) == L and len(named(calls, "q_mlp_forward_")) == L
            assert head == {"gemm_half_q_half"} and "rms_norm" in names
            if sched == "D6" and staged:
                assert 8 < B <= 16          # the 9..16-row wgmma, not the many-row path
        elif sched == "D4":
            assert not dec.fused_attn and not fused and len(ref_attn) == L
            assert len(named(calls, "q_to_fp16_kv")) == L and len(named(calls, "fp16_to_q_kv")) == L
            assert head == {"gemm_half_q_half"} and "rms_norm" in names
        else:
            raise KeyError(sched)
        return
    if kind == "prefill":
        qlens = [a[3] for a, _ in attn1_ex] + [a[3] for a, _ in attn1]
        if sched == "P1":
            assert dec.chained and dec.fused_attn and B == 1
            if staged:
                assert not attn1 and [a[3] for a, _ in attn1_ex] == [8] * L + [3] * L
            else:
                assert not attn1_ex and [a[3] for a, _ in attn1] == [8] * L + [3] * L
                assert [a[0].shape[1] for a, _ in fused] == [8] * L + [3] * L
            assert "gemv_norm" not in names and "gemm_half_q_half_prepared" not in names
        elif sched == "P2":
            assert dec.fused_attn and B == 3
            assert not attn1_ex and [a[2] * a[3] for a, _ in attn1] == [24] * L + [9] * L   # 24 > 16: gemm_big; 9: wgmma
            assert [a[0].shape[1] for a, _ in fused] == [8] * L + [3] * L
        elif sched == "P4":
            assert not dec.fused_attn and not fused and ref_attn and max(qlens) <= 8
            assert len(named(calls, "q_to_fp16_kv")) == len(ref_attn) == len(named(calls, "fp16_to_q_kv"))
        # (prompts of decode schedules run in the decode schedule's flags; their numbers are checked all the same)
        return
    if kind == "rows_q":        # prefill_rows(cache_attn=True); paged_attn_prefill_q is spied by test_gpu_decoder_prefill_q.PrefillSpy
        assert len(attn1) == L and len(named(calls, "paged_attn_prefill_q")) == L and len(named(calls, "q_mlp_forward_rows")) == L
        assert not named(calls, "q_to_fp16_kv") and not named(calls, "fp16_to_q_kv") and not named(calls, "_sdpa_prefill")
        return
    assert kind == "rows"
    assert len(named(calls, "q_to_fp16_kv")) == L and len(named(calls, "fp16_to_q_kv")) == L
    assert len(attn1) == L and len(named(calls, "q_mlp_forward_rows")) == L
    assert len(named(calls, "_sdpa_prefill")) == (L if model._flash_attn_with_kvcache() is None else 0)


# ---- checks of one decoder call, shared by the GPU decoder tests ---------------------------------------------------------------

# rel-L2 of the decoder's output vs the fp64 truth, per schedule: about 2x the worst measured on an H100 (DESIGN.md §3.6)
OUT_TOL = {"D1": 5e-3, "D2": 5e-3, "D3": 5e-3, "D4": 3e-3, "D5": 9e-3, "D6": 1e-2,
           "P1": 5e-3, "P2": 7e-3, "P3": 6e-3, "P4": 4e-3, "L": 6e-3}
# appended cache rows: |unpack(stored) - truth| <= KV_RATIO * |unpack(pack(fp16(truth))) - truth| + KV_SLACK * |truth|
KV_RATIO = 1.1
KV_SLACK = 2e-3
# The fp16 floor of a call: how far the ideal fp16-storage forward (fp16=True) lies from the exact one on the same input.  It is
# <= FLOOR_TYPICAL on almost every input; where the residual stream cancels it is several times larger, and so is any fp16
# implementation's error there (on the hd-128 model some decode steps have a floor of 1-2e-2).  The output bound of a call scales
# by floor / FLOOR_TYPICAL above that, and an appended cache row may be off by FLOOR_RATIO x its own floor.
FLOOR_TYPICAL = 3e-3
FLOOR_RATIO = 3.0


def snapshot(dec):
    c = dec.cache
    return dict(k=[t.cpu().numpy().copy() for t in c.key_states], ks=[t.cpu().numpy().copy() for t in c.key_scales],
                v=[t.cpu().numpy().copy() for t in c.value_states], vs=[t.cpu().numpy().copy() for t in c.value_scales],
                seqlens=c.cache_seqlens.cpu().numpy().copy(), bt=c.block_table.cpu().numpy().copy())


def slots(snap, b, lo, hi):
    from exllamav2_b200.model import PAGE_SIZE
    p = np.arange(lo, hi)
    return snap["bt"][b][p // PAGE_SIZE], p % PAGE_SIZE


def cache_kv(snap, cfg, bits, li, b, lo, hi):
    """Dequantised K and V of sequence b, positions [lo, hi), layer li: [n, KVH, hd] fp64, following the stored page table."""
    import kv_q68
    n, shp = hi - lo, (hi - lo, cfg.num_kv_heads, cfg.head_dim)
    if n == 0:
        return np.zeros(shp), np.zeros(shp)
    pg, r = slots(snap, b, lo, hi)
    kb, vb = kv_q68.widths(bits)
    k = kv_q68.kv_unpack(snap["k"][li][pg, r].reshape(n, -1), snap["ks"][li][pg, r].reshape(n, -1), kb)
    v = kv_q68.kv_unpack(snap["v"][li][pg, r].reshape(n, -1), snap["vs"][li][pg, r].reshape(n, -1), vb)
    return k.astype(np.float64).reshape(shp), v.astype(np.float64).reshape(shp)


def row_err(stored, truth, b):
    """(|stored - truth|, |unpack(pack(fp16(truth))) - truth|, |truth|) per row; rows [n, KVH, hd]."""
    import kv_q68
    t = truth.reshape(truth.shape[0], -1)
    rq = kv_q68.kv_unpack(*kv_q68.kv_pack(t.astype(np.float16), b), b).astype(np.float64)
    s = stored.reshape(t.shape)
    return np.linalg.norm(s - t, axis=1), np.linalg.norm(rq - t, axis=1), np.linalg.norm(t, axis=1)


def as_starts(starts, B: int) -> np.ndarray:
    """Per-sequence first positions of a call: an int array [B], or one int for every sequence."""
    a = np.asarray(starts, dtype=np.int64).reshape(-1)
    return np.full(B, int(a[0]), dtype=np.int64) if a.size == 1 else a


def check_call(dec, truth, sched, kind, ids, out, pre, post, starts, chunk=8, floor_ratio=0.0, poison=None, allow=None, stats=None):
    """What every checked decoder call must satisfy, given the cache snapshots before (pre) and after (post) it and its output
    (decode: logits [B, vocab]; prompt: hidden state [B, T_last, hidden]).  starts: each sequence's position before the call
    (an int array [B], or one int for all); dec.pos, the host's mirror, must have advanced from max(starts):
      (3) cache_seqlens advanced by exactly the tokens fed, per sequence, dec.pos with them, the page table untouched;
      (2a) cache bytes at positions written before the call unchanged;
      (2b) each appended row, dequantised, within KV_RATIO x the format's own quantisation error of the truth row (+ slack,
           or FLOOR_RATIO x that row's fp16 floor);
      (2c) with `poison` (poison_past), every poisoned byte the call did not append into unchanged;
      (1) the output per sequence within OUT_TOL[sched] rel-L2 of the truth, scaled up by floor / FLOOR_TYPICAL where this
          input's fp16 floor is larger than that, and never below floor_ratio x the floor (0: off) or allow[b] (None: off).
    stats: a dict that receives the per-sequence output rel-L2 ("err") and fp16 floor ("floor").
    Returns (worst output rel-L2, worst floor, number of sequences whose bound was scaled)."""
    import kv_q68
    from exl2_oracle import rel_l2
    cfg, bits = dec.cfg, dec.cache.wbits
    B, T = ids.shape
    L = cfg.num_layers
    starts = as_starts(starts, B)
    assert np.array_equal(pre["seqlens"], starts), (pre["seqlens"], starts)
    assert np.array_equal(post["seqlens"], pre["seqlens"] + T), (pre["seqlens"], post["seqlens"], T)
    assert dec.pos == int(starts.max()) + T
    assert np.array_equal(post["bt"], pre["bt"])
    assert np.isfinite(out).all()
    if poison is not None:
        check_poison(poison, post, starts, T)
    kb, vb = kv_q68.widths(bits)
    worst, worst_floor, floored = 0.0, 0.0, 0
    chunks = [(t0, min(chunk, T - t0)) for t0 in range(0, T, chunk)] if kind == "prefill" else [(0, T)]
    for b in range(B):
        pos0 = int(starts[b])
        pg, r = slots(pre, b, 0, pos0)
        for key in ("k", "ks", "v", "vs"):
            for li in range(L):
                assert np.array_equal(post[key][li][pg, r], pre[key][li][pg, r]), f"seq {b} layer {li}: {key} of the past changed"
        for t0, n in chunks:
            start = pos0 + t0
            past = [cache_kv(post, cfg, bits, li, b, 0, start) for li in range(L)]
            pk, pv = [p[0] for p in past], [p[1] for p in past]
            res = truth.forward(ids[b, t0:t0 + n], start, pk, pv)
            res16 = truth.forward(ids[b, t0:t0 + n], start, pk, pv, fp16=True)
            for li in range(L):
                k, v = cache_kv(post, cfg, bits, li, b, start, start + n)
                for got, want, want16, wb, what in ((k, res.k[li], res16.k[li], kb, "K"), (v, res.v[li], res16.v[li], vb, "V")):
                    e, eq, nt = row_err(got, want, wb)
                    floor = np.linalg.norm((want16 - want).reshape(n, -1), axis=1)
                    bad = e > KV_RATIO * eq + np.maximum(KV_SLACK * nt, FLOOR_RATIO * floor)
                    assert not bad.any(), (f"seq {b} layer {li} {what} rows {start + np.flatnonzero(bad)}: error "
                                           f"{e[bad] / nt[bad]} vs quantisation {eq[bad] / nt[bad]}, fp16 floor {floor[bad] / nt[bad]}")
        want, want16 = (res.logits[-1], res16.logits[-1]) if kind == "decode" else (res.hidden, res16.hidden)
        err, floor = rel_l2(out[b], want), rel_l2(want16, want)
        if stats is not None:
            stats.setdefault("err", []).append(err)
            stats.setdefault("floor", []).append(floor)
        bound = max(OUT_TOL[sched] * max(1.0, floor / FLOOR_TYPICAL), floor_ratio * floor, 0.0 if allow is None else allow[b])
        floored += bound > OUT_TOL[sched]
        worst, worst_floor = max(worst, err), max(worst_floor, floor)
        assert err <= bound, (f"{sched} seq {b} (start {pos0}): rel-L2 {err:.3e} vs the fp64 truth (bound {bound:.3e}, "
                              f"fp16 floor {floor:.3e})")
    return worst, worst_floor, floored


# ---- rows past each sequence's length ---------------------------------------------------------------------------------------

# Scales of a poisoned row: codes times scale reach 2^12 before the inverse Hadamard (4-bit codes -8..7 x 2^9, 8-bit codes
# -128..127 x 2^5), so a dequantised element is at most 2^12 and stays finite in fp16 however the rotation sums it.  Against
# a live key of norm ~1 such a row scores hundreds to thousands of nats above (or below) every live row: in each head about
# half of them would take the whole softmax mass if any leaked into a max, a sum or P V.
POISON_SCALE = {4: 2.0 ** 9, 8: 2.0 ** 5}


def poison_rows(rng, shape_q, shape_s, bits):
    """Random codes at the poison scale: (codes uint8 [shape_q], scales fp16 [shape_s])."""
    return rng.integers(0, 256, size=shape_q, dtype=np.uint8), np.full(shape_s, POISON_SCALE[bits], dtype=np.float16)


def poison_past(dec, lens, rng):
    """Overwrite every cache row at a position >= lens[b] in sequence b's pages, and every row of a page no sequence owns, in
    every layer, K and V, with random codes at the poison scale (POISON_SCALE).  Returns the poison: the mask of poisoned
    (page, row) slots and a snapshot of the cache with it in place, for check_poison."""
    import kv_q68
    import torch
    from exllamav2_b200.model import PAGE_SIZE
    c = dec.cache
    kb, vb = kv_q68.widths(c.wbits)
    bt = c.block_table.cpu().numpy()
    mask = np.ones((c.key_states[0].shape[0], PAGE_SIZE), dtype=bool)
    for b, n in enumerate(lens):
        p = np.arange(int(n))
        mask[bt[b][p // PAGE_SIZE], p % PAGE_SIZE] = False
    n = int(mask.sum())
    idx = tuple(torch.from_numpy(a).to(c.key_states[0].device) for a in np.nonzero(mask))
    for li in range(dec.cfg.num_layers):
        for q, s, bits in ((c.key_states[li], c.key_scales[li], kb), (c.value_states[li], c.value_scales[li], vb)):
            pq, ps = poison_rows(rng, (n,) + tuple(q.shape[2:]), (n,) + tuple(s.shape[2:]), bits)
            q[idx] = torch.from_numpy(pq).to(q.device)
            s[idx] = torch.from_numpy(ps).to(s.device)
    return dict(mask=mask, snap=snapshot(dec))


def check_poison(poison, post, starts, T):
    """Every poisoned slot but the ones this call appended into ([start, start + T) of each sequence) holds the poison's bytes;
    the appended slots leave the poison."""
    for b, s in enumerate(starts):
        pg, r = slots(post, b, int(s), int(s) + T)
        poison["mask"][pg, r] = False
    m = poison["mask"]
    for key in ("k", "ks", "v", "vs"):
        for li, (a, w) in enumerate(zip(post[key], poison["snap"][key])):
            assert np.array_equal(a[m].view(np.uint8), w[m].view(np.uint8)), f"layer {li}: a poisoned {key} byte past a length changed"


def graph_matches_eager(dec, ids, on_eager=None):
    """One decode step eagerly, then the same step (same cache state) by graph replay: identical logits and cache bytes.  Leaves
    the decoder as it was, with the graph armed.  on_eager() runs right after the eager step (the caller's branch check)."""
    import torch
    c = dec.cache
    live = (*c.key_states, *c.key_scales, *c.value_states, *c.value_scales, c.cache_seqlens)
    state = [t.clone() for t in live]

    def restore():
        for dst, src in zip(live, state):
            dst.copy_(src)

    g, dec.graph = dec.graph, None
    x = torch.from_numpy(ids).to(c.cache_seqlens.device)
    eager = dec.decode(x).clone()
    eager_cache = snapshot(dec)
    if on_eager is not None:
        on_eager()
    restore()
    dec.pos -= 1
    dec.graph = g
    replay = dec.decode(x).clone()
    replay_cache = snapshot(dec)
    assert torch.equal(eager.view(torch.int16), replay.view(torch.int16)), "graph replay differs from the eager step"
    for key in ("k", "ks", "v", "vs"):
        for a, b in zip(eager_cache[key], replay_cache[key]):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), f"graph replay stored different {key}"
    assert np.array_equal(eager_cache["seqlens"], replay_cache["seqlens"])
    restore()
    dec.pos -= 1


# ---- one un-chained fused decode step (D3 / D6), launch by launch --------------------------------------------------------------

# Per-launch bounds, rel-L2 per sequence against fp64 on the launch's own fp16 inputs: the block entry points' bounds at full
# size (DESIGN.md §3.7: attention block part 1 / part 2, MLP block, head) and the fused attention's (§3.4).
LAUNCH_TOL = {"q_attn_forward_1": 1.5e-3, "paged_attn_decode_q4": 1.6e-3, "q_attn_forward_2": 5e-4, "q_mlp_forward_": 3e-3,
              "rms_norm": 1e-3, "gemm_half_q_half": 5e-4}


def replay_fused_step(dec, ids):
    """One decode step of the fused, un-chained branch (ExLlamaV2Decoder._forward_tokens at q_len 1, then the rms_norm + gemm
    head), issued here launch by launch on the decoder's own handles and cache, the same calls in the same order.  After each
    launch its output is compared with fp64 on that launch's own fp16 inputs: weights from get_weight_tensor_dq(), cached rows
    dequantised by the oracle.  Advances the decoder as decode() would.  Returns {(launch, layer): rel-L2 per sequence [B]}."""
    import torch
    import attn_regimes as ar
    import kv_q68
    from exllamav2_b200 import ext
    from exllamav2_b200.model import PAGE_SIZE
    cfg, c = dec.cfg, dec.cache
    B, H, KVH, hd, eps = dec.batch_size, cfg.num_heads, cfg.num_kv_heads, cfg.head_dim, cfg.norm_eps
    kb, vb = kv_q68.widths(c.wbits)
    f64 = lambda t: t.to(torch.float64)
    W = [l.get_weight_tensor_dq() for l in dec.linears]
    out = {}

    def rel(got, want):
        g, w = f64(got).reshape(B, -1), want.reshape(B, -1)
        return ((g - w).norm(dim=1) / w.norm(dim=1).clamp_min(1e-30)).cpu().numpy()

    def norm(x, w):
        x = f64(x)
        return x / (x * x).mean(-1, keepdim=True).add(eps).sqrt() * f64(w)

    sl = c.cache_seqlens.cpu().numpy().copy()
    bt = c.block_table.cpu().numpy()
    pos = torch.as_tensor(sl, device=dec.device)
    cos, sin = f64(dec.cos)[pos, :hd // 2][:, None, :], f64(dec.sin)[pos, :hd // 2][:, None, :]

    def rope(t, heads):
        t = t.view(B, heads, hd)
        l, r = t[..., :hd // 2], t[..., hd // 2:]
        return torch.cat([l * cos - r * sin, r * cos + l * sin], -1)

    x = dec.embed[torch.as_tensor(ids, device=dec.device).view(-1)].contiguous().view(B, 1, -1)
    q, k, v = dec.q, dec.k, dec.v
    ao = dec.attn_out
    for li, L in enumerate(dec.layers):
        wq, wk, wv, wo, wg, wu, wd = W[7 * li:7 * li + 7]
        x0 = x.clone()
        ext.q_attn_forward_1(L.attn, x, B, 1, -1, c.cache_seqlens, q, k, v, dec.sin, dec.cos)
        xn = norm(x0.view(B, -1), L.input_norm)
        want = [rope(xn @ f64(wq), H), rope(xn @ f64(wk), KVH), xn @ f64(wv)]
        out[("q_attn_forward_1", li)] = np.max([rel(t, w) for t, w in zip((q, k, v), want)], axis=0)
        # attention: the cached rows [0, seqlen) as the oracle dequantises them, then the unquantised new row
        qn, kn, vn = (t.view(B, 1, -1, hd).cpu().numpy() for t in (q, k, v))
        snap = snapshot(dec)
        Kr = [ar.gather_rows(snap["k"][li], snap["ks"][li], bt, b, int(sl[b]), kb, PAGE_SIZE) for b in range(B)]
        Vr = [ar.gather_rows(snap["v"][li], snap["vs"][li], bt, b, int(sl[b]), vb, PAGE_SIZE) for b in range(B)]
        ext.paged_attn_decode_q4(q.view(B, 1, H, hd), k.view(B, 1, KVH, hd), v.view(B, 1, KVH, hd), c.key_states[li],
                                 c.key_scales[li], c.value_states[li], c.value_scales[li], c.cache_seqlens, c.block_table,
                                 ao.view(B, 1, H, hd), 1.0 / math.sqrt(hd), wbits=c.wbits)
        want = torch.as_tensor(ar.attention_truth(qn, kn, vn, Kr, Vr, sl, 1.0 / math.sqrt(hd)), device=dec.device)
        out[("paged_attn_decode_q4", li)] = rel(ao, want)
        x0, a0 = x.clone(), ao.clone()
        ext.q_attn_forward_2(L.attn, x, ao, B, 1)
        out[("q_attn_forward_2", li)] = rel(x, f64(x0).view(B, -1) + f64(a0).view(B, -1) @ f64(wo))
        x0 = x.clone()
        ext.q_mlp_forward_(L.mlp, x)
        xn = norm(x0.view(B, -1), L.post_norm)
        g = xn @ f64(wg)
        out[("q_mlp_forward_", li)] = rel(x, f64(x0).view(B, -1) + (g / (1 + torch.exp(-g)) * (xn @ f64(wu))) @ f64(wd))
    c.cache_seqlens.add_(1)
    dec.pos += 1
    ext.rms_norm(x.view(B, -1), dec.final_norm, dec.xn, eps)
    out[("rms_norm", -1)] = rel(dec.xn, norm(x.view(B, -1), dec.final_norm))
    ext.gemm_half_q_half(dec.xn, dec.lm_head.q_handle, dec.logits, False)
    out[("gemm_half_q_half", -1)] = rel(dec.logits, f64(dec.xn) @ f64(W[-1]))
    torch.cuda.synchronize()
    return out
