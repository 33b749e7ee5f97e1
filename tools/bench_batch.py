"""Batched decode sweep: today's un-chained schedule against the chained one, B sequences per step, each step one CUDA graph.

    python tools/bench_batch.py [--batches 1,8,9,12,16,17,24,32,48,64] [--steps 64] [--runs 3] [--prompt 128] [--out DIR]

7B preset (llama2-7b-4.0bpw), Q4 cache, a prompt of --prompt tokens per sequence.  For every B the two schedules are captured
in the same process and timed alternately (--runs rounds of --steps replays each):
  * "unchained": dec.chained = False (the decoder's schedule for 9..16 sequences, and for 17+ before the wide tiles);
  * "chained":   the chained step; at 9..16 sequences forced through _forward_tokens_chained + the prepared head.
Prints one JSON line per (B, schedule): tok/s median [min, max], ms/step, kernel launches per step (torch.profiler, one
replay), algorithmic bytes per step (packed weights once + K/V cache rows read + activations) and GB/s, rel-L2 between the two
schedules' logits on the same state, and the card's name, power limit and max SM clock read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:          # the numbers are reported without it, and say so
        return f"not read ({e})"


def step_fn(dec, chained):
    from exllamav2_b200 import ext as ext_c

    def forced():
        torch.index_select(dec.embed, 0, dec.ids.view(-1), out=dec.x.view(dec.batch_size, -1))
        dec._forward_tokens_chained(dec.x, dec.q, dec.k, dec.v, dec.attn_out, 1, head=True)
        ext_c.gemm_half_q_half_prepared(dec.lm_head.q_handle, dec.logits, True, dec.cfg.norm_eps)

    if chained and not dec._chains(dec.batch_size):
        return forced
    return dec._decode_step


def capture(dec, fn):
    saved = dec.cache.cache_seqlens.clone()
    s = torch.cuda.Stream(dec.device)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        fn()
        torch.cuda.synchronize()
        dec.cache.cache_seqlens.copy_(saved)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            fn()
    torch.cuda.synchronize()
    dec.cache.cache_seqlens.copy_(saved)
    return g


def launches(g):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        g.replay()
        torch.cuda.synchronize()
    return sum(1 for e in p.events() if e.device_type.name == "CUDA" and "Memcpy" not in e.name and "Memset" not in e.name)


def step_bytes(dec, B, ctx):
    from exllamav2_b200 import ext as ext_c
    cfg = dec.cfg
    w = sum(ext_c.q_matrix_info(l.q_handle)["packed_bytes"] for l in dec.linears)
    kv_row = cfg.num_kv_heads * cfg.head_dim
    bits = dec.cache.wbits
    kv = cfg.num_layers * B * ctx * 2 * kv_row * (bits / 8 + 2 / 32)     # codes + one fp16 scale per 32 values
    act = cfg.num_layers * B * 2 * (4 * cfg.hidden_size + 2 * cfg.intermediate_size) + B * cfg.vocab_size * 2
    return w + kv + act


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,9,12,16,17,24,32,48,64")
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--prompt", type=int, default=128)
    ap.add_argument("--model", default="llama2-7b-4.0bpw")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_batch needs a GPU"
    from exllamav2_b200.model import PRESETS, ExLlamaV2Decoder
    dev = "cuda:0"
    info = card()
    rows = []
    for B in [int(b) for b in args.batches.split(",")]:
        cache_len = (args.prompt + args.steps * args.runs * 2 + 16 + 255) // 256 * 256
        dec = ExLlamaV2Decoder(PRESETS[args.model](), device=dev, seed=0, batch_size=B, cache_len=cache_len, cache_bits=4)
        g = torch.Generator().manual_seed(B)
        prompt = torch.randint(0, dec.cfg.vocab_size, (B, args.prompt), generator=g).to(dev)
        dec.prefill_rows(prompt)
        dec.ids.copy_(prompt[:, -1:])
        torch.cuda.synchronize()
        graphs, logits = {}, {}
        for sched in ("unchained", "chained"):
            dec.chained = sched == "chained"
            graphs[sched] = capture(dec, step_fn(dec, sched == "chained"))
        saved = dec.cache.cache_seqlens.clone()
        for sched in ("unchained", "chained"):       # the same state through both: the logits must agree
            dec.cache.cache_seqlens.copy_(saved)
            graphs[sched].replay()
            torch.cuda.synchronize()
            logits[sched] = dec.logits.float().clone()
        dec.cache.cache_seqlens.copy_(saved)
        rel = (torch.linalg.norm(logits["chained"] - logits["unchained"]) / torch.linalg.norm(logits["unchained"])).item()
        for sched in graphs:       # warm-up
            for _ in range(4):
                graphs[sched].replay()
        torch.cuda.synchronize()
        times = {s: [] for s in graphs}
        for _ in range(args.runs):
            for sched in ("unchained", "chained"):
                dec.cache.cache_seqlens.copy_(saved)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(args.steps):
                    graphs[sched].replay()
                torch.cuda.synchronize()
                times[sched].append((time.perf_counter() - t0) / args.steps)
        ctx = args.prompt + 1
        nbytes = step_bytes(dec, B, ctx)
        for sched in ("unchained", "chained"):
            ts = times[sched]
            tok = sorted(B / t for t in ts)
            r = dict(B=B, schedule=sched, tok_s=statistics.median(tok), tok_s_min=tok[0], tok_s_max=tok[-1],
                     ms_step=statistics.median(ts) * 1e3, launches=launches(graphs[sched]), bytes_step=int(nbytes),
                     gb_s=nbytes / statistics.median(ts) / 1e9, rel_l2_vs_other=rel, card=info,
                     chained_by_rule=dec._chains(B) if sched == "chained" else False)
            rows.append(r)
            print(json.dumps(r), flush=True)
        del graphs
        dec.unload()
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_batch.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
