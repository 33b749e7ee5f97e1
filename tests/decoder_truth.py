"""fp64 restatement of one ExLlamaV2Decoder call (exllamav2_b200/model.py), teacher-forced on the K/V the decoder stored.

Plain math throughout, not the fp16-rounded oracle ops: embedding row -> per layer [RMSNorm -> q/k/v = xn W -> NeoX RoPE at the
token's absolute position -> causal GQA attention with scale 1/sqrt(hd) -> o_proj + residual -> RMSNorm -> SiLU(gate) * up ->
down + residual] -> final RMSNorm -> LM head.

Positions before the call's first token come from the caller (the decoder's own cache bytes, dequantised): the truth of a call
is then a continuous function of its inputs, so a kernel that is a little off cannot hide behind a free-running sequence that
drifted across a quantisation step.  The call's own tokens enter attention unquantised, as they do in the fused kernel.
"""
from __future__ import annotations

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
