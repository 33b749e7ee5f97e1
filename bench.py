#!/usr/bin/env python
"""bench.py -- decode tokens/s (bs=1) of a Llama-2-7B-shaped EXL2 ~4.0 bpw model on the sm_90a (H100) hot path,
with the q_gemm path's achieved HBM GB/s against the measured roofline.  BASELINE.json metric / configs[2].

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--model PRESET] [--dump-outputs DIR]

A "step" is one decode token: embedding -> 32 x (Q4-KV unpack, RMSNorm+QKV+RoPE, paged attention, Q4-KV pack,
O-proj+residual, RMSNorm+gate|up+silu*mul, down+residual) -> RMSNorm -> lm_head.  Weights are synthetic tensors in the
reference's on-disk EXL2 format (no network), resident in HBM; 3.3 GB of packed weights per token >> 50 MB L2, so no
L2 flush is needed between steps ("inputs_exceed_l2").

--dump-outputs DIR writes what the last timed step returned to its caller: for decode DIR/logits.npy (float32 [1, vocab])
and DIR/next_token.npy (float64 [1, 1], the on-device argmax fed to the next step; with --gpus N rank 0 writes the
all-gathered logits), for --mode prefill DIR/hidden.npy (float32 [16, prompt_len, hidden], the final hidden states of the
timed many-row pass).  Weights, prompts and synthetic cache rows are seeded, so two builds run with the same arguments
can be compared output for output.

JSON keys (one line on stdout):
  value / ms_per_step   device-timed (CUDA events) over K graph replays, next token chosen by an on-device argmax
  e2e                   same metric through the public API with HOST buffers: pinned token id -> H2D, decode,
                        fp16 logits -> pinned host (D2H), host argmax, every step
  roofline              the dominant kernel (gemv_kernel): sum of algorithmic bytes of every linear of the model
                        / device time of exactly those launches replayed back to back, vs MEASURED_PEAKS.json hbm_gbs
  cpu_baseline          oracle/exl2_cpu.c (the CPU port of the reference's q_gemm) on the host cores, bounded sample
  --impl reference      the CPU arm alone (the reference has no CPU q_gemm; its CUDA extension is timed separately by
                        tools/microbench.py --ref and reported under "reference_cuda_ext" when oracle/_ref is present)
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "decode tokens/sec (bs=1) Llama2-7B EXL2-4.0bpw"       # the default --model; other presets are named in config.workload
UNIT = "tokens/s"


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------

def dump_outputs(outdir: str, **arrays) -> None:
    """--dump-outputs: each array as outdir/<name>.npy, float32 (float64 for token ids)."""
    import numpy as np
    os.makedirs(outdir, exist_ok=True)
    for name, t in arrays.items():
        a = t.detach().cpu()
        a = a.double() if not a.is_floating_point() else a.float()
        np.save(os.path.join(outdir, f"{name}.npy"), a.numpy())


def measured_peaks() -> tuple[float, str]:
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        try:
            return float(json.load(open(p))["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
        except Exception:
            pass
    return 3350.0, "fallback (H100 SXM data sheet 3.35 TB/s, not measured)"


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled every 200 ms while the timed region runs."""

    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index: int = 0):
        self.index, self.samples, self._stop, self._t = index, [], threading.Event(), None

    def _run(self):
        while not self._stop.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--id={self.index}", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits"],
                                     capture_output=True, text=True, timeout=5).stdout.strip()
                if out:
                    self.samples.append([s.strip() for s in out.split(",")])
            except Exception:
                pass
            self._stop.wait(0.2)

    def __enter__(self):
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()
        return self

    def __exit__(self, *a):
        self._stop.set()
        self._t.join(timeout=6)

    def summary(self) -> dict:
        sm = sorted(int(float(s[0])) for s in self.samples if s and s[0].replace(".", "").isdigit())
        reasons = []
        for name, col in (("hw_slowdown", 3), ("hw_thermal_slowdown", 4), ("sw_thermal_slowdown", 5), ("sw_power_cap", 6)):
            if any(len(s) > col and s[col].lower().startswith("active") for s in self.samples):
                reasons.append(name)
        mx = next((int(float(s[1])) for s in self.samples if len(s) > 1 and s[1].replace(".", "").isdigit()), None)
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx, "reasons": reasons, "samples": len(self.samples)}


# Shapes / bit plans of the reference arm: COPIED from exllamav2_b200/model.py PRESETS on purpose -- the reference arm must not
# import the product package (its process would map libexl2b200.so)
REF_ARM_CONFIGS = {
    "llama2-7b-4.0bpw": dict(hidden=4096, inter=11008, heads=32, kv_heads=32, head_dim=128, layers=32, vocab=32000,
                             attn=((5, 4), (0.1, 0.9), 128),
                             mlp=[((5, 4), (0.1, 0.9), 128), ((5, 4), (0.1, 0.9), 128), ((4, 3), (0.1, 0.9), 128), ((5, 4), (0.1, 0.9), 128)],
                             head_bits=6),
    "llama2-7b-4bit-g128": dict(hidden=4096, inter=11008, heads=32, kv_heads=32, head_dim=128, layers=32, vocab=32000,
                                attn=((4,), (1.0,), 128), mlp=[((4,), (1.0,), 128)], head_bits=6),
    "tinyllama-1.1b-4.0bpw": dict(hidden=2048, inter=5632, heads=32, kv_heads=4, head_dim=64, layers=22, vocab=32000,
                                  attn=((4,), (1.0,), 128), mlp=[((4,), (1.0,), 128)], head_bits=6),
}
_CPU_MATS: dict = {}


def cpu_port_baseline(model: str, budget_s: float = 12.0, n_layers: int = 3) -> dict:
    """Time oracle/exl2_cpu.c (fused CPU dequant-GEMV over the checkpoint layout) on the seven matrices of `n_layers` DISTINCT
    decoder layers (different bit plans where the model mixes them), all host threads; extrapolate to tokens/s by bytes."""
    import numpy as np
    # torchrun exports OMP_NUM_THREADS=1 for its workers: this arm is a host-cores baseline, use all of them
    ncpu = os.cpu_count() or 1
    os.environ["OMP_NUM_THREADS"] = str(ncpu)
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import oracle_c
    import synth
    lib = oracle_c.load()
    try:
        lib.omp_set_num_threads(ncpu)          # libgomp is linked into libexl2_cpu.so; overrides an inherited OMP_NUM_THREADS
    except AttributeError:
        pass
    threads = lib.exl2_cpu_threads()
    c = REF_ARM_CONFIGS[model]
    rng = np.random.default_rng(0)
    hid, inter, H, KVH, hd = c["hidden"], c["inter"], c["heads"], c["kv_heads"], c["head_dim"]

    def rand_exl2(K, N, plan):
        bits, prop, gs = plan
        gp = synth.group_plan(K, list(bits), list(prop), gs)
        G = len(gp)
        qg = np.zeros((2 * G,), dtype=np.int16)
        row = 0
        for i, (b, rows) in enumerate(gp):
            qg[2 * i], qg[2 * i + 1] = b, row
            row += rows * b // 32
        return dict(qw=rng.integers(0, 2**32, size=(row, N), dtype=np.uint32), qs=rng.integers(0, 2**32, size=(G, N // 8), dtype=np.uint32),
                    smax=rng.uniform(0.002, 0.015, size=(G,)).astype(np.float16).view(np.uint16), qg=qg,
                    perm=rng.permutation(K).astype(np.uint16), K=K, N=N, G=G, R=row)

    key = (model, n_layers)
    if key not in _CPU_MATS:
        layers = []
        for li in range(n_layers):
            mp = c["mlp"][(li + 1) % len(c["mlp"])]          # li = 1 lands on the [4,3] plan of the 4.0 bpw preset
            layers.append([rand_exl2(hid, H * hd, c["attn"]), rand_exl2(hid, KVH * hd, c["attn"]), rand_exl2(hid, KVH * hd, c["attn"]),
                           rand_exl2(H * hd, hid, c["attn"]), rand_exl2(hid, inter, mp), rand_exl2(hid, inter, mp), rand_exl2(inter, hid, mp)])
        _CPU_MATS[key] = layers
    layers = _CPU_MATS[key]
    ins = [[rng.normal(size=(m["K"],)).astype(np.float32) for m in mats] for mats in layers]
    outs = [[np.empty((m["N"],), dtype=np.float32) for m in mats] for mats in layers]

    def one_pass():
        ts = []
        for mats, ia, oa in zip(layers, ins, outs):
            t0 = time.perf_counter()
            for m, a, y in zip(mats, ia, oa):
                oracle_c.exl2_gemv_prepared(lib, m, a, y)
            ts.append(time.perf_counter() - t0)
        return ts

    one_pass()
    per_layer: list[float] = []
    t_start = time.perf_counter()
    n = 0
    while True:
        per_layer += one_pass()
        n += 1
        if time.perf_counter() - t_start > budget_s or n >= 30:
            break
    per_layer.sort()
    t_layer = per_layer[len(per_layer) // 2]                          # median layer time
    layer_w = sum(m["qw"].nbytes for mats in layers for m in mats) / len(layers)
    head_w = c["hidden"] * c["vocab"] * c["head_bits"] // 8
    t_token = t_layer * c["layers"] + t_layer * head_w / layer_w
    return {"value": 1.0 / t_token, "unit": UNIT, "cores": threads, "kind": "port",
            "sample": f"oracle/exl2_cpu.c fused dequant-GEMV on {len(layers)} distinct decoder layers (7 matrices each, {layer_w / 1e6:.0f} MB packed "
                      f"per layer), {n} passes, median layer x{c['layers']} layers + head by bytes",
            "ms_per_layer": {"min": per_layer[0] * 1e3, "median": t_layer * 1e3, "max": per_layer[-1] * 1e3}}


# ---------------------------------------------------------------------------------------------------------------------
# arms
# ---------------------------------------------------------------------------------------------------------------------

def run_reference(args, rank, world):
    """Reference arm: the reference's CPU implementation of the path on the host cores.  The reference has no CPU
    q_gemm (SURVEY.md 8d), so this is the oracle port (kind "port"), each step = one bounded sample over three layers.
    Imports nothing of the product package."""
    if rank != 0:
        return
    vals = []
    for i in range(args.warmup + args.steps):
        r = cpu_port_baseline(args.model, budget_s=max(0.25, 90.0 / max(1, args.warmup + args.steps)))
        if i >= args.warmup:
            vals.append(r)
    vs = sorted(x["value"] for x in vals)
    v = vs[len(vs) // 2]
    cb = dict(vals[-1])
    cb["value"] = v
    cb["spread"] = {"min": vs[0], "median": v, "max": vs[-1]}
    line = {"impl": "reference", "metric": METRIC, "value": v, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": 1e3 / v, "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "fp32 accumulate over int weights",
            "data": "synthetic", "config": {"workload": f"{args.model} decode bs=1 (CPU port of q_gemm, weights only)"},
            "cpu_baseline": cb, "e2e": {"value": v, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)


def run_ours(args, rank, world):
    import torch
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200.model import PRESETS, ExLlamaV2Decoder
    if world > 1:
        from exllamav2_b200 import tensor_p
        return tensor_p.run_bench(args, rank, world, METRIC, UNIT)

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    cfg = PRESETS[args.model]()
    t_build = time.time()
    ctx = args.context if args.context > 0 else args.prompt_len
    need = ctx + 2 * (max(3, args.warmup) + args.steps) + 16
    dec = ExLlamaV2Decoder(cfg, dev, seed=0, batch_size=1, cache_len=max(1024, (need + 255) // 256 * 256))
    torch.cuda.synchronize()
    t_build = time.time() - t_build
    g = torch.Generator(device="cpu").manual_seed(0)
    prompt = torch.randint(0, cfg.vocab_size, (1, args.prompt_len), generator=g).to(dev)
    if args.context > 0:
        # synthetic cache rows (random nibbles, scales of a unit-variance row): the decode step's cost does not depend on their values
        gd = torch.Generator(device=dev).manual_seed(1)
        for li in range(cfg.num_layers):
            for t in (dec.cache.key_states[li], dec.cache.value_states[li]):
                t.copy_(torch.randint(0, 256, t.shape, dtype=torch.uint8, device=dev, generator=gd))
            for t in (dec.cache.key_scales[li], dec.cache.value_scales[li]):
                t.fill_(0.35)
        dec.cache.cache_seqlens.fill_(args.context)
        dec.pos = args.context
        dec.ids.copy_(prompt[:, -1:])
    else:
        dec.prefill(prompt)
    torch.cuda.synchronize()

    # graph: decode step + on-device greedy pick feeding the next step (fully device-resident loop)
    def step_with_argmax():
        dec._decode_step()
        torch.argmax(dec.logits, dim=-1, keepdim=True, out=dec.ids)

    saved = dec.cache.cache_seqlens.clone()
    s = torch.cuda.Stream(dev)
    with torch.cuda.stream(s):
        step_with_argmax()
        torch.cuda.synchronize()
        dec.cache.cache_seqlens.copy_(saved)
        l0 = ext_c.launch_count()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            step_with_argmax()
        launches_per_step = ext_c.launch_count() - l0
    torch.cuda.synchronize()
    dec.cache.cache_seqlens.copy_(saved)
    dec.ids.copy_(prompt[:, -1:])

    if os.environ.get("EXL2B_PROFILE"):
        # ncu --profile-from-start off: capture exactly two eager decode steps (launch list / --set full)
        torch.cuda.synchronize()
        torch.cuda.profiler.start()
        for _ in range(2):
            step_with_argmax()
        torch.cuda.synchronize()
        torch.cuda.profiler.stop()
        print(json.dumps({"profiled_steps": 2}))
        return
    W, K = max(3, args.warmup), args.steps
    assert ctx + 2 * (W + K) + 8 < dec.cache.max_seq_len
    for _ in range(W):
        graph.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with ClockSampler(0) as clk:
        torch.cuda.synchronize()
        e0.record()
        for _ in range(K):
            graph.replay()
        e1.record()
        torch.cuda.synchronize()
    ms_total = e0.elapsed_time(e1)
    ms_per_step = ms_total / K
    assert bool(torch.isfinite(dec.logits).all()), "decode produced non-finite logits"
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, logits=dec.logits, next_token=dec.ids)
    value = 1000.0 / ms_per_step

    # ---- parity of the TIMED path: the same token through the chained launches (what the graph replays) and through the
    #      reference's un-chained op sequence (q_attn_forward_1 incl. rope_, attention, q_attn_forward_2, q_mlp_forward_, rms_norm
    #      + gemm_half_q_half), same cache state; tests/test_gpu_row_blocks.py pins each of those ops to the oracle at <= 1e-3
    parity = {}
    try:
        saved2 = dec.cache.cache_seqlens.clone()
        tok = dec.ids.clone()
        dec._decode_step()
        la = dec.logits.float().clone()
        dec.cache.cache_seqlens.copy_(saved2)
        dec.ids.copy_(tok)
        was = dec.chained
        dec.chained = False
        dec._decode_step()
        dec.chained = was
        lb = dec.logits.float().clone()
        dec.cache.cache_seqlens.copy_(saved2)
        dec.ids.copy_(tok)
        parity["timed_vs_unchained_logits_rel_l2"] = float((torch.linalg.norm(la - lb) / torch.linalg.norm(lb)).item())
        parity["attn_status"] = ext_c.paged_attn_status(dev)
    except Exception as e:      # noqa: BLE001
        parity["error"] = str(e)[:200]

    # ---- e2e: host buffers every step --------------------------------------------------------------------------
    dec.capture()     # plain decode graph (no device argmax)
    ids_host = torch.zeros((1, 1), dtype=torch.long).pin_memory()
    logits_host = torch.empty((1, cfg.vocab_size), dtype=torch.half).pin_memory()
    ids_host[0, 0] = int(dec.ids[0, 0].item())
    for _ in range(3):
        dec.ids.copy_(ids_host, non_blocking=True)
        dec.graph.replay()
        logits_host.copy_(dec.logits, non_blocking=True)
        torch.cuda.synchronize()
        ids_host[0, 0] = int(torch.argmax(logits_host.float(), dim=-1)[0])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(K):
        dec.ids.copy_(ids_host, non_blocking=True)
        dec.graph.replay()
        logits_host.copy_(dec.logits, non_blocking=True)
        torch.cuda.synchronize()
        ids_host[0, 0] = int(torch.argmax(logits_host.float(), dim=-1)[0])
    t_e2e = (time.perf_counter() - t0) / K
    e2e = {"value": 1.0 / t_e2e, "unit": UNIT, "h2d_bytes_per_step": 8, "d2h_bytes_per_step": cfg.vocab_size * 2,
           "ms_per_step": t_e2e * 1e3}

    # ---- roofline of the dominant kernel: exactly the model's GEMV launches, back to back ------------------------
    # (the chained decode loop of exllamav2_b200/model.py minus the attention kernel: Q|K|V, O, gate|up, down per layer
    #  + lm_head -- same handles, same fused epilogues, same buffers as the timed decode step)
    def gemv_only():
        if dec.chained and dec.fused_attn:
            dec._forward_tokens_chained(dec.x, dec.q, dec.k, dec.v, dec.attn_out, 1, head=True, gemv_only=True)
            if dec.row_gemv:
                ext_c.gemv_norm(dec.x.view(1, -1), dec.lm_head.q_handle, dec.final_norm, cfg.norm_eps, dec.logits, prepared=True)
            else:
                ext_c.gemm_half_q_half_prepared(dec.lm_head.q_handle, dec.logits, True, cfg.norm_eps)
        else:
            for L in dec.layers:
                ext_c.q_attn_forward_1(L.attn, dec.x, 1, 1, -1, dec.cache.cache_seqlens, dec.q, dec.k, dec.v, dec.sin, dec.cos)
                ext_c.q_attn_forward_2(L.attn, dec.x, dec.attn_out, 1, 1)
                ext_c.q_mlp_forward_(L.mlp, dec.x)
            ext_c.gemm_half_q_half(dec.xn, dec.lm_head.q_handle, dec.logits, False)

    dec.x.normal_()
    with torch.cuda.stream(s):
        gemv_only()
        torch.cuda.synchronize()
        l0 = ext_c.launch_count()
        g2 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g2, stream=s):
            gemv_only()
        n_launch_roof = ext_c.launch_count() - l0
    n_gemv = 4 * cfg.num_layers + 1
    for _ in range(3):
        g2.replay()
    torch.cuda.synchronize()
    e0.record()
    R = 20
    for _ in range(R):
        g2.replay()
    e1.record()
    torch.cuda.synchronize()
    ms_gemv = e0.elapsed_time(e1) / R
    peak, peak_src = measured_peaks()
    achieved = dec.weight_bytes / (ms_gemv * 1e-3) / 1e9
    roofline = {"bound": "hbm", "kernel": "gemv_i8_kernel" if dec.row_gemv else "gemm_tc_kernel", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                "peak_source": peak_src, "algorithmic_bytes_per_token": dec.weight_bytes,
                "gemv_launches_per_token": n_gemv, "avg_launch_us": ms_gemv * 1e3 / n_gemv,
                "note": f"{n_launch_roof} launches ({n_gemv} dequant-GEMMs + their prep/rope launches, if any) replayed back to back in one CUDA graph, CUDA events"}

    cpu = cpu_port_baseline(args.model) if (not args.no_cpu and args.model in REF_ARM_CONFIGS) else None
    # ---- the real competitor: the unmodified reference extension (oracle/_ref) on the same synthetic model, same GPU, same
    #      process, in the reference's own per-layer op sequence (oracle/ref_decoder.py); outside every timed region of ours
    ref_ext = None
    if not args.no_ref_ext:
        try:
            del graph, g2
            dec.graph = None
            sys.path.insert(0, os.path.join(ROOT, "oracle"))
            import ref_decoder
            ref_ext = ref_decoder.time_reference_decode(cfg, prompt_len=args.prompt_len, steps=min(K, 64), warmup=W, device="cuda:0")
        except Exception as e:      # noqa: BLE001
            ref_ext = {"unavailable": str(e)[:300]}
    line = {
        "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": 1, "steps": K, "warmup": W, "ms_per_step": ms_per_step,
        "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "fp16 (int2-8 weights, fp32 accumulate)",
        "data": "synthetic",
        "config": {"workload": f"{cfg.name} single-stream decode, " + (f"{args.context}-position synthetic context" if args.context > 0 else f"{args.prompt_len}-token prompt") + ", Q4 KV cache, bs=1",
                   "l2": f"inputs_exceed_l2 ({dec.weight_bytes / 1e9:.2f} GB of weights per step)", "weight_bytes": dec.weight_bytes, "build_s": round(t_build, 1),
                   "quant_plan": {"attn": str(cfg.plan.attn), "mlp (cycled over layers)": str(cfg.plan.mlp), "head": str(cfg.plan.head)}},
        "clocks": clk.summary(), "e2e": e2e, "gpu_launches": int(launches_per_step * K), "launches_per_step": int(launches_per_step),
        "roofline": roofline, "cpu_baseline": cpu, "parity": parity, "reference_cuda_ext": ref_ext,
    }
    print(json.dumps(line), flush=True)


def run_prefill(args):
    """--mode prefill (BASELINE configs[2] "bs=16 prefill"): 16 sequences x prompt_len tokens through every layer in ONE weight pass
    per matrix (many-row path: reconstruct + dense tensor-core GEMM) vs the 8-row chunks the decode kernels would need."""
    import torch
    from exllamav2_b200.model import PRESETS, ExLlamaV2Decoder
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    cfg = PRESETS[args.model]()
    B, T = 16, args.prompt_len
    dec = ExLlamaV2Decoder(cfg, dev, seed=0, batch_size=B, cache_len=1024)
    g = torch.Generator(device="cpu").manual_seed(0)
    prompt = torch.randint(0, cfg.vocab_size, (B, T), generator=g).to(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn, reps):
        ts = []
        for i in range(reps + 1):
            dec.cache.cache_seqlens.zero_()
            dec.pos = 0
            torch.cuda.synchronize()
            e0.record()
            out = fn(prompt)
            e1.record()
            torch.cuda.synchronize()
            if i:
                ts.append(e0.elapsed_time(e1))
        return sorted(ts)[len(ts) // 2], out
    ms_rows, x_rows = timed(dec.prefill_rows, args.steps)
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, hidden=x_rows)
    ms_chunk, x_chunk = timed(lambda p: dec.prefill(p, chunk=8), 1)
    # same prompt, two schedules: the hidden state of the last chunk must agree (Q4 cache in the loop: loose tolerance)
    a, b = x_rows[:, -8:].float(), x_chunk.float()
    rel = float((torch.linalg.norm(a - b) / torch.linalg.norm(b)).item())
    from exllamav2_b200 import model as _m
    line = {"metric": "prefill tokens/sec (bs=16) Llama2-7B EXL2-4.0bpw", "value": B * T / (ms_rows * 1e-3), "unit": UNIT, "n_gpus": 1,
            "ms_per_step": ms_rows, "higher_is_better": True, "dtype": "fp16 (int2-8 weights dequantised to fp16, fp32 accumulate)", "data": "synthetic",
            "config": {"workload": f"{cfg.name} prompt processing, {B} sequences x {T} tokens = {B * T} rows, Q4 KV cache",
                       "attention": "flash_attn_with_kvcache" if _m._flash_attn_with_kvcache() is not None else "torch SDPA"},
            "chunked_8_rows": {"ms_per_step": ms_chunk, "value": B * T / (ms_chunk * 1e-3), "note": "same prompt through the 8-row decode kernels (round-1 path)"},
            "hidden_rel_l2_rows_vs_chunked": rel,
            "hidden_note": "one pass attends the chunk's own K/V in fp16 (like the reference: flash-attn on the fp16 temp, then store_kv_state), 8-row chunks "
                           "attend earlier chunks through the 4-bit cache: the two schedules differ by the cache's quantisation error, amplified over 32 "
                           "random-weight layers; per-op parity of the many-row path is tests/test_gpu_linear.py / test_gpu_row_blocks.py"}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--model", default="llama2-7b-4.0bpw")
    ap.add_argument("--prompt-len", type=int, default=128)
    ap.add_argument("--context", type=int, default=0,
                    help="decode at this context length: the Q4 cache is filled with synthetic rows up to N positions (no prompt pass); 0 = run the prompt")
    ap.add_argument("--mode", default="decode", choices=["decode", "prefill"])
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--no-ref-ext", action="store_true", help="skip the reference-extension leg (oracle/_ref on the same GPU)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write what the last timed step returned as DIR/<name>.npy (decode: logits, next token; prefill: hidden states)")
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    if args.dump_outputs and args.impl != "ours":
        ap.error("--dump-outputs writes this library's outputs (--impl ours)")
    rank = int(os.environ.get("RANK", "0"))
    if args.impl == "reference":
        return run_reference(args, rank, world)
    if args.mode == "prefill":
        return run_prefill(args) if rank == 0 else None
    return run_ours(args, rank, world)


if __name__ == "__main__":
    main()
