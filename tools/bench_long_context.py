#!/usr/bin/env python
"""Decode attention just below and just above the capacity where one score buffer stops fitting shared memory, measured in
one process with the two capacities alternating.

    python tools/bench_long_context.py [--bits 4] [--steps 32] [--reps 5] [--layers 4] [--out FILE.json]

For each shape -- the 7B preset at B = 8 (32 heads, hd 128), the 70B preset at B = 1 (64 heads over 8), TinyLlama at B = 8
(32 heads over 4, hd 64) -- two capacities: the largest that takes the single-pass plan (tests/attn_long_plan.py
largest_fit) and one page more, which walks each CTA's positions in passes (csrc/attn_q4.cu attn_q4_passes_kernel).  Every
sequence is full (seqlen = capacity - 1 for attention alone; capacity - 2 * (steps + 8) for decode), synthetic cache rows
(random bytes, fixed scales, as bench.py --context).
  * attention alone: the fused kernel, CUDA events around --steps launches; algorithmic bytes per launch (DESIGN.md §7):
    per cached position and kv head hd * (KB + VB) / 8 + 2 * 2 * hd / 32;
  * decode tok/s: the preset with its first --layers layers (the caches of a full 7B at B = 8 would not fit twice), the step
    captured as one CUDA graph, CUDA events over --steps replays, tokens = B per step.
Medians over --reps rounds; within a round the two capacities run back to back.  The card name and power limit are read in
the same process.  Writes nothing into the tree (stdout, or --out)."""
import argparse
import dataclasses
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import attn_long_plan as alp  # noqa: E402
from bench_kvcache import WIDTHS, card, median  # noqa: E402
from exllamav2_b200 import ext as ext_c  # noqa: E402
from exllamav2_b200.model import PAGE_SIZE, PRESETS, ExLlamaV2Decoder  # noqa: E402

SHAPES = [("llama2-7b-4.0bpw", 8), ("llama2-70b-2.5bpw", 1), ("tinyllama-1.1b-4.0bpw", 8)]
DEV = "cuda:0"


def attn_bytes(cfg, B, seqlen, bits):
    kb, vb = WIDTHS[bits]
    hd = cfg.head_dim
    return B * seqlen * cfg.num_kv_heads * (hd * (kb + vb) // 8 + 2 * 2 * hd // 32)


class AttnCase:
    """One layer's cache at capacity `cap` for B full sequences, and the inputs of one launch."""

    def __init__(self, cfg, B, cap, bits):
        kb, vb = WIDTHS[bits]
        H, KVH, hd = cfg.num_heads, cfg.num_kv_heads, cfg.head_dim
        pages = B * cap // PAGE_SIZE
        g = torch.Generator(device=DEV).manual_seed(cap)
        self.k = torch.randint(0, 256, (pages, PAGE_SIZE, KVH, hd * kb // 8), dtype=torch.uint8, device=DEV, generator=g)
        self.v = torch.randint(0, 256, (pages, PAGE_SIZE, KVH, hd * vb // 8), dtype=torch.uint8, device=DEV, generator=g)
        self.ks = torch.full((pages, PAGE_SIZE, KVH, hd // 32), 0.35, dtype=torch.half, device=DEV)
        self.vs = torch.full_like(self.ks, 0.35)
        self.bt = torch.arange(pages, dtype=torch.int32, device=DEV).view(B, -1)
        self.sl = torch.full((B,), cap - 1, dtype=torch.int32, device=DEV)
        self.q = torch.randn((B, 1, H, hd), dtype=torch.half, device=DEV)
        self.kn = torch.randn((B, 1, KVH, hd), dtype=torch.half, device=DEV)
        self.vn = torch.randn((B, 1, KVH, hd), dtype=torch.half, device=DEV)
        self.out = torch.empty_like(self.q)
        self.scale, self.bits = 1.0 / math.sqrt(hd), bits

    def launch(self):
        ext_c.paged_attn_decode_q4(self.q, self.kn, self.vn, self.k, self.ks, self.v, self.vs, self.sl, self.bt, self.out,
                                   self.scale, wbits=self.bits)

    def time(self, n):
        self.launch()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            self.launch()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3 / n


def make_decoder(cfg, B, cap, bits, steps):
    dec = ExLlamaV2Decoder(cfg, DEV, seed=0, batch_size=B, cache_len=cap, cache_bits=bits)
    gd = torch.Generator(device=DEV).manual_seed(1)
    for li in range(cfg.num_layers):
        for t in (dec.cache.key_states[li], dec.cache.value_states[li]):
            t.copy_(torch.randint(0, 256, t.shape, dtype=torch.uint8, device=DEV, generator=gd))
        for t in (dec.cache.key_scales[li], dec.cache.value_scales[li]):
            t.fill_(0.35)
    ctx = cap - 2 * (steps + 8)
    dec.cache.cache_seqlens.fill_(ctx)
    dec.pos = ctx
    dec.ids.fill_(7)
    torch.cuda.synchronize()
    dec.capture()
    return dec


def time_steps(dec, steps, B):
    saved = dec.cache.cache_seqlens.clone()
    for _ in range(4):
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
    return 1000.0 * steps * B / e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bits", type=int, default=4, choices=(4, 6, 8))
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--layers", type=int, default=4, help="decoder layers of the preset kept for decode tok/s (0: skip decode)")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    result = {"card": card(), "cache_bits": args.bits, "steps": args.steps, "reps": args.reps, "layers": args.layers, "rows": []}
    print(json.dumps(result["card"]), flush=True)
    for model, B in SHAPES:
        cfg = PRESETS[model]()
        below = alp.largest_fit(args.bits, cfg.head_dim, cfg.num_heads, B)
        caps = (below, below + PAGE_SIZE)
        plans = [alp.long_plan(args.bits, cfg.head_dim, cfg.num_heads, B, 1, c) for c in caps]
        assert not plans[0]["passes"] and plans[1]["passes"]
        att = {c: AttnCase(cfg, B, c, args.bits) for c in caps}
        dcfg = dataclasses.replace(cfg, num_layers=args.layers, max_seq_len=max(cfg.max_seq_len, caps[1]))
        decs = {c: make_decoder(dcfg, B, c, args.bits, args.steps) for c in caps} if args.layers > 0 else {}
        us = {c: [] for c in caps}
        tok = {c: [] for c in caps}
        for _ in range(args.reps):
            for c in caps:                           # the two capacities alternate within every round
                us[c].append(att[c].time(args.steps))
                if decs:
                    tok[c].append(time_steps(decs[c], args.steps, B))
        for c, p in zip(caps, plans):
            sec = median(us[c])
            nb = attn_bytes(cfg, B, c - 1, args.bits)
            row = {"model": model, "batch": B, "capacity": c, "passes": p["passes"], "pass_len": p["pass_len"],
                   "nsplit": p["nsplit"], "attn_us_per_launch": round(sec * 1e6, 2), "attn_bytes": nb,
                   "attn_gb_s": round(nb / sec / 1e9, 1), "attn_us_min_max": [round(min(us[c]) * 1e6, 2), round(max(us[c]) * 1e6, 2)]}
            if decs:
                row.update(tok_s=round(median(tok[c]), 2), tok_s_min_max=[round(min(tok[c]), 2), round(max(tok[c]), 2)])
            result["rows"].append(row)
            print(json.dumps(row), flush=True)
        for d in decs.values():
            d.unload()
        del att, decs
        torch.cuda.empty_cache()
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
