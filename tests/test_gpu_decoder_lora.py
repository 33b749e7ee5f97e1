"""The decoder with LoRA adapters (ExLlamaV2Decoder.load_lora / set_loras) against an fp64 Llama forward with the adapters' terms,
teacher-forced on the K/V cache bytes the decoder itself stored (tests/decoder_truth.py: the same per-call checks and bounds as
the adapter-free decoder tests; a step with adapters runs the un-chained block forms, so its bounds are those of the un-chained
schedules: D3 at batch 1, D6 above).

Batch-1 decode eager and replayed from a captured graph, batch-8 ragged decode (per-sequence lengths, rows past each length
poisoned), prefill, prefill_rows on both attention paths; Q4 and Q8 caches.  And: after set_loras([]) the 7B preset's step is the
chained 161-launch step again, with logits byte-identical to a decoder that never loaded an adapter."""

import numpy as np
import pytest
import torch

import decoder_truth as dt

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED = 3
F64 = np.float64


class LoraTruth(dt.TruthModel):
    """TruthModel.forward with y_P += (in_P A) B for every active adapter on projection P.  fp16=True rounds the same stored
    intermediates TruthModel.forward rounds (the adapted projections included), so the fp16 floor check_call derives from it is
    the adapted model's own."""

    def __init__(self, base: dt.TruthModel, adapters: list):
        self.__dict__.update(base.__dict__)
        self.adapters = adapters          # per layer {projection: [(A, B), ...]}

    def _d(self, li, p, inp):
        return sum(((inp @ a) @ b for a, b in self.adapters[li].get(p, [])), np.zeros((inp.shape[0], 1)))

    def forward(self, ids, start, past_k, past_v, fp16=False):
        ids = np.asarray(ids).reshape(-1)
        T = ids.shape[0]
        H, KVH, hd = self.H, self.KVH, self.hd
        r = dt._round16 if fp16 else (lambda a: a)
        pos = start + np.arange(T)
        x = self.embed[ids].copy()
        ks, vs = [], []
        for li, L in enumerate(self.layers):
            xn = r(dt.rms_norm(x, L.input_norm, self.eps))
            q = r(dt.rope_neox(r(xn @ L.wq + self._d(li, "q_proj", xn)).reshape(T, H, hd), self.sin, self.cos, pos))
            k = r(dt.rope_neox(r(xn @ L.wk + self._d(li, "k_proj", xn)).reshape(T, KVH, hd), self.sin, self.cos, pos))
            v = r((xn @ L.wv + self._d(li, "v_proj", xn)).reshape(T, KVH, hd))
            ks.append(k)
            vs.append(v)
            kc = np.concatenate([np.asarray(past_k[li], dtype=F64), k])
            vc = np.concatenate([np.asarray(past_v[li], dtype=F64), v])
            o = r(dt.attention(q, kc, vc, start).reshape(T, H * hd))
            x = r(x + r(o @ L.wo + self._d(li, "o_proj", o)))
            xn = r(dt.rms_norm(x, L.post_norm, self.eps))
            g = r(xn @ L.wg + self._d(li, "gate_proj", xn))
            u = r(xn @ L.wu + self._d(li, "up_proj", xn))
            a = r(dt.silu(g) * u)
            x = r(x + r(a @ L.wd + self._d(li, "down_proj", a)))
        logits = dt.rms_norm(x, self.final_norm, self.eps) @ self.head
        return dt.CallTruth(hidden=x, logits=logits, k=ks, v=vs)


def _cfg(model):
    from exllamav2_b200.model import PRESETS, LlamaConfig
    if model == "hd128":
        return LlamaConfig("test-hd128-gqa", 1024, 2816, 8, 4, 128, 2, 1024, max_seq_len=512, plan=PRESETS["test-small"]().plan)
    return PRESETS["test-small"]()


def _decoder(B, bits, model="small"):
    from exllamav2_b200.model import ExLlamaV2Decoder
    dec = ExLlamaV2Decoder(_cfg(model), device=DEV, seed=SEED, batch_size=B, cache_len=512, cache_bits=bits)
    a = dec.load_lora(16, seed=1)                                           # every projection
    b = dec.load_lora(64, targets=("q_proj", "v_proj"), scaling=0.5, seed=2)  # the common PEFT target
    dec.set_loras([a, b])
    return dec


def _truth(dec):
    cfg = dec.cfg
    h = lambda t: t.float().cpu().numpy().astype(F64)
    W = [h(l.get_weight_tensor_dq()) for l in dec.linears]
    layers = [dt.TruthLayer(h(L.input_norm), h(L.post_norm), *W[7 * li:7 * li + 7]) for li, L in enumerate(dec.layers)]
    base = dt.TruthModel(layers, h(dec.final_norm), W[-1], h(dec.embed), h(dec.sin), h(dec.cos), cfg.num_heads, cfg.num_kv_heads,
                         cfg.head_dim, cfg.norm_eps)
    ads = []
    for li in range(cfg.num_layers):
        d = {}
        for key in dec.lora_ids:
            for p, (a, b) in dec.loras[key][li].items():
                d.setdefault(p, []).append((h(a), h(b)))
        ads.append(d)
    t = LoraTruth(base, ads)
    # the adapters matter: the adapter-free forward is far from this one
    ids = np.arange(3)
    zero = [np.zeros((0, cfg.num_kv_heads, cfg.head_dim))] * cfg.num_layers
    from exl2_oracle import rel_l2
    assert rel_l2(base.forward(ids, 0, zero, zero).logits, t.forward(ids, 0, zero, zero).logits) > 0.02
    return t


def _check(dec, truth, sched, kind, ids, run, poison=None):
    pre = dt.snapshot(dec)
    starts = pre["seqlens"].astype(np.int64)
    out = run(torch.from_numpy(ids).to(DEV)).float().cpu().numpy()
    torch.cuda.synchronize()
    worst, floor, _ = dt.check_call(dec, truth, sched, kind, ids, out, pre, dt.snapshot(dec), starts, poison=poison)
    print(f"TRUTH lora {sched} Q{dec.cache.wbits} {kind} B={ids.shape[0]} T={ids.shape[1]}: out rel-L2 {worst:.3e} floor {floor:.3e}")
    return worst


def _ids(B, T, V, seed):
    return np.random.default_rng(seed).integers(0, V, size=(B, T)).astype(np.int64)


@pytest.mark.parametrize("bits", [4, 8])
def test_decode_b1_eager_and_graph(bits):
    dec = _decoder(1, bits)
    truth = _truth(dec)
    V = dec.cfg.vocab_size
    _check(dec, truth, "P1", "prefill", _ids(1, 11, V, 1), lambda x: dec.prefill(x, 8))
    for s in range(3):
        _check(dec, truth, "D3", "decode", _ids(1, 1, V, 10 + s), dec.decode)
    dec.capture()
    dt.graph_matches_eager(dec, _ids(1, 1, V, 20))
    for s in range(3):
        _check(dec, truth, "D3", "decode", _ids(1, 1, V, 30 + s), dec.decode)
    dec.set_loras(dec.lora_ids)
    assert dec.graph is None                  # set_loras drops the captured step


@pytest.mark.parametrize("bits", [4, 8])
def test_decode_b8_ragged(bits):
    dec = _decoder(8, bits)
    truth = _truth(dec)
    V = dec.cfg.vocab_size
    rng = np.random.default_rng(bits)
    lens = [9, 1, 0, 5, 9, 3, 7, 2]
    prompt = np.repeat(rng.integers(0, V, size=(1, max(lens))), 8, axis=0).astype(np.int64)
    dec.prefill_rows(torch.from_numpy(prompt).to(DEV))
    torch.cuda.synchronize()
    dec.cache.cache_seqlens.copy_(torch.tensor(lens, dtype=torch.int32, device=DEV))
    dec.pos = max(lens)
    poison = dt.poison_past(dec, lens, rng)
    for s in range(2):
        _check(dec, truth, "D6", "decode", _ids(8, 1, V, 40 + s), dec.decode, poison=poison)
        poison = None
    dec.capture()
    dt.graph_matches_eager(dec, _ids(8, 1, V, 50))


@pytest.mark.parametrize("cache_attn", [False, True])
@pytest.mark.parametrize("bits", [4, 8])
def test_prefill_rows(cache_attn, bits):
    dec = _decoder(2, bits, "hd128" if cache_attn else "small")
    truth = _truth(dec)
    V = dec.cfg.vocab_size
    _check(dec, truth, "P3", "rows", _ids(2, 20, V, 60), lambda x: dec.prefill_rows(x, cache_attn=cache_attn))
    _check(dec, truth, "P3", "rows", _ids(2, 7, V, 61), lambda x: dec.prefill_rows(x, cache_attn=cache_attn))
    _check(dec, truth, "P2", "prefill", _ids(2, 11, V, 62), lambda x: dec.prefill(x, 8))
    _check(dec, truth, "D6", "decode", _ids(2, 1, V, 63), dec.decode)


def test_clearing_returns_to_the_chained_step():
    """7B preset: with adapters cleared the step is the chained 161-launch step, and its logits are byte-identical to those of a
    decoder that never loaded an adapter."""
    from exllamav2_b200 import ext
    from exllamav2_b200.model import PRESETS, ExLlamaV2Decoder
    cfg = PRESETS["llama2-7b-4.0bpw"]()
    ids = torch.tensor([[17]], device=DEV)
    plain = ExLlamaV2Decoder(cfg, device=DEV, seed=0, cache_len=512)
    want = plain.decode(ids).clone()
    plain.unload()
    del plain
    torch.cuda.empty_cache()
    dec = ExLlamaV2Decoder(cfg, device=DEV, seed=0, cache_len=512)
    assert torch.equal(dec.decode(ids).view(torch.int16), want.view(torch.int16))     # (first use builds plans and buffers)
    dec.cache.cache_seqlens.zero_()
    dec.pos = 0
    key = dec.load_lora(16, seed=1)
    dec.set_loras([key])
    torch.cuda.synchronize()
    n0 = ext.launch_count()
    adapted = dec.decode(ids).clone()
    torch.cuda.synchronize()
    n_adapted = ext.launch_count() - n0
    assert not torch.equal(adapted, want)
    dec.cache.cache_seqlens.zero_()
    dec.pos = 0
    dec.set_loras([])
    n0 = ext.launch_count()
    got = dec.decode(ids).clone()
    torch.cuda.synchronize()
    assert ext.launch_count() - n0 == 161
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))
    print(f"7B step launches: {n_adapted} with rank-16 adapters on every projection, 161 without")
    dec.unload_lora(key)
    assert dec.loras == {} and dec.lora_ids == []
    dec.unload()
