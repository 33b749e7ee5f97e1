"""Prompt attention of one layer, two ways, on the GPU (JSON lines on stdout):

  (a) what ExLlamaV2Decoder.prefill_rows runs by default: get_kv_state (q_to_fp16_kv of the whole live cache) + attention on
      the fp16 temp (flash_attn_with_kvcache if it imports and runs, else torch SDPA, _sdpa_prefill) + store_kv_state;
  (b) paged_attn_prefill_q (csrc/attn_prefill.cu): attention straight over the quantised cache, append in the same launch.

Each point alternates the two paths over several rounds after warming both up and reports the median ms of each by CUDA events,
the algorithmic FLOPs 4 hd H sum(causal pairs) as TFLOP/s and as a share of the 989 TFLOP/s dense-fp16 data-sheet rate of the
H100 SXM, and the rel-L2 between (a) and (b).  Then the whole prefill_rows call both ways at bench.py's prefill workload on the 7B
preset.  The card's name and power limit are printed first.

    python tools/bench_prefill_attn.py [--rounds 5] [--reps 10] [--wbits 4]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_FP16 = 989e12


def causal_pairs(seqlens, T):
    return sum(T * s + T * (T + 1) // 2 for s in seqlens)


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q)


def point(H, KVH, hd, B, T, seqlen, wbits, rounds, reps):
    import torch
    from exllamav2_b200 import ext
    from exllamav2_b200 import model as m
    dev = torch.device("cuda:0")
    cfg = m.LlamaConfig("attn-only", H * hd, 1, H, KVH, hd, 1, 1)
    cache_len = (seqlen + T + m.PAGE_SIZE - 1) // m.PAGE_SIZE * m.PAGE_SIZE
    cache = m.CACHE_CLASSES[wbits](cfg, B, cache_len, dev)
    g = torch.Generator(device=dev).manual_seed(0)
    for t in (cache.key_states[0], cache.value_states[0]):
        t.copy_(torch.randint(0, 256, t.shape, generator=g, device=dev, dtype=torch.int32).to(torch.uint8))
    for t, z in ((cache.key_scales[0], 8 if wbits == 4 else 128), (cache.value_scales[0], 128 if wbits == 8 else 8)):
        t.copy_((torch.rand(t.shape, generator=g, device=dev) * 0.6 + 0.4) * (2.0 / z))
    cache.cache_seqlens.fill_(seqlen)
    q = torch.randn((B, T, H, hd), generator=g, device=dev).half()
    k = (0.3 * torch.randn((B, T, KVH, hd), generator=g, device=dev)).half()
    v = (0.3 * torch.randn((B, T, KVH, hd), generator=g, device=dev)).half()
    scale = 1.0 / math.sqrt(hd)
    fa = m._flash_attn_with_kvcache()
    out_b = torch.empty_like(q)

    def path_a(use_fa=True):
        tk, tv = cache.get_kv_state(0)
        if fa is not None and use_fa:
            o = fa(q=q, k=k, v=v, k_cache=tk, v_cache=tv, cache_seqlens=cache.cache_seqlens, block_table=cache.block_table,
                   causal=True, softmax_scale=scale)
        else:
            o = m._sdpa_prefill(q, k, v, tk, tv, cache, hd)
        cache.store_kv_state(0, T)
        return o

    def path_b():
        ext.paged_attn_prefill_q(q, k, v, cache.key_states[0], cache.key_scales[0], cache.value_states[0], cache.value_scales[0],
                                 cache.cache_seqlens, cache.block_table, out_b, scale, wbits=wbits)
        return out_b

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    oa, ob = path_a().float(), path_b().float()          # warm-up of both, and the outputs compared
    torch.cuda.synchronize()
    rel = float((torch.linalg.norm(oa - ob) / torch.linalg.norm(oa)).item())
    ta, tb = [], []
    for _ in range(rounds):
        ta.append(timed(path_a))
        tb.append(timed(path_b))
    ms_a, ms_b = sorted(ta)[len(ta) // 2], sorted(tb)[len(tb) // 2]
    flops = 4 * hd * H * causal_pairs([seqlen] * B, T)
    extra = {}
    if fa is not None:          # what prefill_rows runs where flash-attn is not installed, timed the same way
        path_a(False)
        ts = []
        for _ in range(rounds):
            ts.append(timed(lambda: path_a(False)))
            timed(path_b)
        ms_s = sorted(ts)[len(ts) // 2]
        extra = dict(ms_a_sdpa=round(ms_s, 4), speedup_vs_sdpa=round(ms_s / ms_b, 3))
    res = dict(kind="attention", H=H, KVH=KVH, hd=hd, B=B, T=T, seqlen=seqlen, wbits=wbits,
               a_path="flash_attn_with_kvcache" if fa is not None else "torch SDPA (_sdpa_prefill)",
               ms_a=round(ms_a, 4), ms_b=round(ms_b, 4), speedup=round(ms_a / ms_b, 3), gflop=round(flops / 1e9, 3),
               tflops_a=round(flops / ms_a / 1e9, 2), tflops_b=round(flops / ms_b / 1e9, 2),
               share_of_989_b=round(flops / (ms_b * 1e-3) / PEAK_FP16, 4), rel_l2_a_vs_b=rel, **extra)
    del cache
    torch.cuda.empty_cache()
    return res


def whole_call(rounds):
    """prefill_rows both ways at bench.py's prefill workload: 7B preset, 16 sequences x 128 tokens, cache 1024, Q4."""
    import torch
    from exllamav2_b200.model import PRESETS, ExLlamaV2Decoder, _flash_attn_with_kvcache
    dev = torch.device("cuda:0")
    cfg = PRESETS["llama2-7b-4.0bpw"]()
    B, T = 16, 128
    dec = ExLlamaV2Decoder(cfg, dev, seed=0, batch_size=B, cache_len=1024)
    prompt = torch.randint(0, cfg.vocab_size, (B, T), generator=torch.Generator(device="cpu").manual_seed(0)).to(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def once(cache_attn):
        dec.cache.cache_seqlens.zero_()
        dec.pos = 0
        torch.cuda.synchronize()
        e0.record()
        x = dec.prefill_rows(prompt, cache_attn=cache_attn)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), x.float()

    _, xa = once(False)
    _, xb = once(True)
    rel = float((torch.linalg.norm(xa - xb) / torch.linalg.norm(xa)).item())
    ta, tb = [], []
    for _ in range(rounds):
        ta.append(once(False)[0])
        tb.append(once(True)[0])
    ms_a, ms_b = sorted(ta)[len(ta) // 2], sorted(tb)[len(tb) // 2]
    dec.unload()
    return dict(kind="prefill_rows", preset=cfg.name, B=B, T=T,
                default_attention="flash_attn_with_kvcache" if _flash_attn_with_kvcache() is not None else "torch SDPA",
                ms_default=round(ms_a, 3), ms_cache_attn=round(ms_b, 3),
                tokens_per_s_default=round(B * T / ms_a * 1e3, 1), tokens_per_s_cache_attn=round(B * T / ms_b * 1e3, 1),
                rel_l2_hidden=rel)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--wbits", type=int, default=4)
    ap.add_argument("--no-whole-call", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_prefill_attn needs a GPU")
    print(json.dumps(dict(kind="card", **card())), flush=True)
    points = [(32, 32, 128, 1, T, s) for T in (512, 2048) for s in (0, 4096, 16384 - T)]
    points += [(64, 8, 128, 1, 2048, 4096), (32, 32, 128, 16, 128, 0)]
    for p in points:
        print(json.dumps(point(*p, args.wbits, args.rounds, args.reps)), flush=True)
    if not args.no_whole_call:
        print(json.dumps(whole_call(args.rounds)), flush=True)


if __name__ == "__main__":
    main()
