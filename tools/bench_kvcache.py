#!/usr/bin/env python
"""Decode speed and attention bandwidth of the Q4, Q6 and Q8 K/V caches, measured in one process with the formats alternating.

    python tools/bench_kvcache.py [--steps 64] [--reps 5] [--out FILE.json]

  * whole-step tok/s: the 7B preset (llama2-7b-4.0bpw), batch 1, the decode step captured as ONE CUDA graph (as bench.py), timed
    with CUDA events over --steps replays; after a 128-token prompt and at synthetic contexts of 4096 and 16384 positions (random
    cache bytes, fixed scales, as bench.py --context);
  * attention alone: the fused decode-attention kernel over all 32 layers' caches in turn (so the working set is far larger than
    L2), CUDA events around --steps rounds.  Algorithmic bytes per launch, from the shapes: per cached position and kv head
    hd * (KB + VB) / 8 bytes of elements + 2 * 2 * hd / 32 bytes of scales.
Each number is the median over --reps rounds; within a round the three formats run back to back.  The card name and power limit
are read in the same process and written to the output.  Writes nothing into the tree (stdout, or --out)."""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from exllamav2_b200 import ext as ext_c  # noqa: E402
from exllamav2_b200.model import PRESETS, ExLlamaV2Decoder  # noqa: E402

BITS = (4, 6, 8)
WIDTHS = {4: (4, 4), 6: (8, 4), 8: (8, 8)}


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20)
        pl, clk = (x.strip() for x in r.stdout.strip().split(","))
        info["power_limit_w"], info["max_sm_clock_mhz"] = float(pl), float(clk)
    except Exception as e:      # noqa: BLE001
        info["power_limit_w"] = f"unavailable ({e!r})"
    return info


def make_decoder(cfg, bits, ctx, steps):
    need = ctx + 2 * (8 + steps) + 16
    dec = ExLlamaV2Decoder(cfg, "cuda:0", seed=0, batch_size=1, cache_len=max(1024, (need + 255) // 256 * 256), cache_bits=bits)
    g = torch.Generator(device="cpu").manual_seed(0)
    prompt = torch.randint(0, cfg.vocab_size, (1, 128), generator=g).cuda()
    if ctx > 128:
        gd = torch.Generator(device="cuda:0").manual_seed(1)
        for li in range(cfg.num_layers):
            for t in (dec.cache.key_states[li], dec.cache.value_states[li]):
                t.copy_(torch.randint(0, 256, t.shape, dtype=torch.uint8, device="cuda:0", generator=gd))
            for t in (dec.cache.key_scales[li], dec.cache.value_scales[li]):
                t.fill_(0.35)
        dec.cache.cache_seqlens.fill_(ctx)
        dec.pos = ctx
        dec.ids.copy_(prompt[:, -1:])
    else:
        dec.prefill(prompt)
    torch.cuda.synchronize()
    dec.capture()
    return dec


def time_steps(dec, steps):
    saved = dec.cache.cache_seqlens.clone()
    for _ in range(8):
        dec.graph.replay()
    torch.cuda.synchronize()
    dec.cache.cache_seqlens.copy_(saved)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        dec.graph.replay()
    e1.record()
    torch.cuda.synchronize()
    dec.cache.cache_seqlens.copy_(saved)
    return 1000.0 * steps / e0.elapsed_time(e1)


def time_attention(dec, ctx, rounds):
    """Seconds per launch of the attention kernel alone, every layer's cache in turn, at context `ctx`."""
    cfg, c = dec.cfg, dec.cache
    H, KVH, hd = cfg.num_heads, cfg.num_kv_heads, cfg.head_dim
    q = torch.randn((1, 1, H, hd), dtype=torch.half, device="cuda:0")
    k = torch.randn((1, 1, KVH, hd), dtype=torch.half, device="cuda:0")
    v = torch.randn((1, 1, KVH, hd), dtype=torch.half, device="cuda:0")
    out = torch.empty_like(q)
    sl = torch.full((1,), ctx, dtype=torch.int32, device="cuda:0")

    def one_round():
        for li in range(cfg.num_layers):
            ext_c.paged_attn_decode_q4(q, k, v, c.key_states[li], c.key_scales[li], c.value_states[li], c.value_scales[li], sl,
                                       c.block_table, out, 1.0 / math.sqrt(hd), wbits=c.wbits)
    one_round()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(rounds):
        one_round()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / (rounds * cfg.num_layers)


def attn_bytes(cfg, ctx, bits):
    kb, vb = WIDTHS[bits]
    hd = cfg.head_dim
    return ctx * cfg.num_kv_heads * (hd * (kb + vb) // 8 + 2 * 2 * hd // 32)


def median(xs):
    s = sorted(xs)
    return s[len(s) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    cfg = PRESETS["llama2-7b-4.0bpw"]()
    result = {"card": card(), "model": cfg.name, "batch": 1, "steps": args.steps, "reps": args.reps, "decode": [], "attention": []}
    for ctx in (128, 4096, 16384):
        decs = {bits: make_decoder(cfg, bits, ctx, args.steps) for bits in BITS}
        tok = {bits: [] for bits in BITS}
        att = {bits: [] for bits in BITS}
        for _ in range(args.reps):
            for bits in BITS:                       # formats alternate within every round
                tok[bits].append(time_steps(decs[bits], args.steps))
            if ctx > 128:
                for bits in BITS:
                    att[bits].append(time_attention(decs[bits], ctx, max(2, args.steps // 8)))
        for bits in BITS:
            row = {"context": ctx, "cache_bits": bits, "tok_s": round(median(tok[bits]), 2),
                   "tok_s_min": round(min(tok[bits]), 2), "tok_s_max": round(max(tok[bits]), 2)}
            result["decode"].append(row)
            print(json.dumps(row), flush=True)
            if ctx > 128:
                sec = median(att[bits])
                nb = attn_bytes(cfg, ctx, bits)
                arow = {"context": ctx, "cache_bits": bits, "us_per_launch": round(sec * 1e6, 2), "bytes_per_launch": nb,
                        "gb_s": round(nb / sec / 1e9, 1)}
                result["attention"].append(arow)
                print(json.dumps(arow), flush=True)
        for d in decs.values():
            d.unload()
        del decs
        torch.cuda.empty_cache()
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
