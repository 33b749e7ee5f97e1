"""What LoRA adapters cost the decoder: tok/s of the whole step captured as one CUDA graph, with and without adapters.

    python tools/bench_lora.py [--model llama2-7b-4.0bpw] [--steps 64] [--warmup 8] [--rounds 5] [--out DIR]

Configurations, alternated within one process round by round so that they see the same machine: no adapter; rank 16 on q and v
(the common PEFT target); rank 16 on all seven projections; rank 64 on all seven -- each also on the un-chained schedule
(`dec.chained = False`, the "-unchained" rows), which is what a step with adapters ran before batch-1 steps could chain them,
and what steps of more than one row with adapters still run.  Workloads: batch-1 and batch-8 decode
(ExLlamaV2Decoder.decode replaying the captured step), and prefill_rows of 16 sequences x 128 tokens (not captured: it
allocates its activations per call).  Per configuration: tok/s as median [min, max] over the rounds, the library's launches per
step (eager), the adapter bytes a token reads on top of the weights (A and B of every active projection, once per step / batch),
and the LoRA kernels' time per step from torch.profiler in a separate, un-timed pass of eager steps (a kernel's time there
runs from its first CTA's start: with programmatic dependent launch that includes waiting for its predecessor; run with
EXL2B_NO_PDL=lora for the kernels' own time).  The card and its power limit
(read-only nvidia-smi query) are printed beside the numbers.  The last line is one JSON object with all of it."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from exllamav2_b200 import ext  # noqa: E402
from exllamav2_b200.model import PRESETS, ExLlamaV2Decoder  # noqa: E402

# name -> (adapter: (rank, targets) or None, chained schedule allowed).  "unchained": no adapter on the un-chained schedule; the
# "-unchained" adapter rows beside their chained ones show what the schedule is worth with adapters
_QV, _ALL = ("q_proj", "v_proj"), ExLlamaV2Decoder.LORA_TARGETS
CONFIGS = {"none": (None, True), "unchained": (None, False),
           "qv-r16": ((16, _QV), True), "qv-r16-unchained": ((16, _QV), False),
           "all-r16": ((16, _ALL), True), "all-r16-unchained": ((16, _ALL), False),
           "all-r64": ((64, _ALL), True), "all-r64-unchained": ((64, _ALL), False)}


def card() -> str:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def adapter_bytes(dec, ids) -> int:
    """bytes of A and B over every layer and active projection: what one step reads on top of the weights"""
    return sum(a.numel() * 2 + b.numel() * 2 for key in ids for layer in dec.loras[key] for a, b in layer.values())


def lora_kernel_us(fn, steps: int) -> float:
    """summed device time of the LoRA kernels per call of fn, from torch.profiler (eager launches)"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    tot = sum(e.device_time_total for e in prof.key_averages() if "lora_kernel" in e.key)
    return tot / steps


def bench_decode(cfg, B: int, args) -> dict:
    # A handle takes at most EXL2B_LORA_MAX_RANK stacked ranks per stage, so the configurations are not registered together: each
    # is loaded, captured and unloaded in turn.  Its graph holds the adapter list by value (the LoRA launches' parameters), so
    # it replays the configuration it was captured with as long as the adapter tensors live (kept here).
    dec = ExLlamaV2Decoder(cfg, batch_size=B, cache_len=1024)
    ids = torch.randint(0, cfg.vocab_size, (B, 1), device="cuda")
    graphs, keep, res = {}, [], {}
    start = dec.cache.cache_seqlens.clone()

    def reset():
        dec.cache.cache_seqlens.copy_(start)
        dec.pos = 0

    for i, (name, (c, chained)) in enumerate(CONFIGS.items()):
        key = dec.load_lora(c[0], targets=c[1], seed=i) if c else None
        dec.set_loras([key] if key else [])
        dec.chained = chained
        torch.cuda.synchronize()
        n0 = ext.launch_count()
        dec.decode(ids)
        torch.cuda.synchronize()
        launches = ext.launch_count() - n0
        reset()
        us = lora_kernel_us(lambda: dec.decode(ids), 8) if key else 0.0
        reset()
        dec.capture()
        graphs[name] = dec.graph
        ab = adapter_bytes(dec, [key]) if key else 0
        res[name] = {"launches_per_step": launches, "adapter_bytes_per_token": ab // B, "lora_kernel_us_per_step": us, "tok_s": []}
        dec.chained = True
        if key:
            keep.append(dec.loras[key])
            dec.unload_lora(key)
    for _ in range(args.rounds):
        for name in CONFIGS:
            dec.graph = graphs[name]
            reset()
            for _ in range(args.warmup):
                dec.decode(ids)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                dec.decode(ids)
            e1.record()
            torch.cuda.synchronize()
            res[name]["tok_s"].append(B * args.steps / (e0.elapsed_time(e1) / 1000.0))
    dec.graph = None
    graphs.clear()
    dec.unload()
    return res


def bench_prefill_rows(cfg, B: int, T: int, args) -> dict:
    dec = ExLlamaV2Decoder(cfg, batch_size=B, cache_len=(T + 255) // 256 * 256)
    ids = torch.randint(0, cfg.vocab_size, (B, T), device="cuda")
    res = {name: {"tok_s": []} for name in CONFIGS}

    def run():
        dec.cache.cache_seqlens.zero_()
        dec.pos = 0
        dec.prefill_rows(ids, cache_attn=True)

    for r in range(args.rounds):
        for i, (name, (c, chained)) in enumerate(CONFIGS.items()):
            key = dec.load_lora(c[0], targets=c[1], seed=i) if c else None
            dec.set_loras([key] if key else [])
            dec.chained = chained          # (prefill_rows never chains: the same as "none")
            run()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            res[name]["tok_s"].append(B * T / (e0.elapsed_time(e1) / 1000.0))
            if r == 0:
                res[name]["lora_kernel_us_per_call"] = lora_kernel_us(run, 2) if key else 0.0
            if key:
                dec.unload_lora(key)
    dec.unload()
    return res


def summary(res: dict) -> dict:
    for r in res.values():
        xs = r.pop("tok_s")
        r["tok_s"] = {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}
    return res


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--model", default="llama2-7b-4.0bpw", choices=sorted(PRESETS))
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lora.py measures on the GPU; none is available")
    cfg = PRESETS[args.model]()
    out = {"card": card(), "model": args.model, "steps": args.steps, "rounds": args.rounds}
    for B in (1, 8):
        out[f"decode_b{B}"] = summary(bench_decode(cfg, B, args))
        torch.cuda.empty_cache()
    out["prefill_rows_16x128"] = summary(bench_prefill_rows(cfg, 16, 128, args))
    print(f"card: {out['card']}")
    for wl in ("decode_b1", "decode_b8", "prefill_rows_16x128"):
        for name, r in out[wl].items():
            t = r["tok_s"]
            extra = " ".join(f"{k}={v:.1f}" if isinstance(v, float) else f"{k}={v}" for k, v in r.items() if k != "tok_s")
            print(f"{wl:22s} {name:17s} {t['median']:9.1f} tok/s [{t['min']:.1f}, {t['max']:.1f}]  {extra}")
    line = json.dumps(out)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_lora.json"), "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
