#!/usr/bin/env python
"""GEMV micro-benchmark: cycles enough distinct matrices that the weights never sit in L2 (methodology of the
reference's tests/test_gemv.py:81-128) and reports achieved algorithmic GB/s for our library and, when
oracle/_ref is built, for the unmodified reference extension on the same GPU.

    python tools/microbench.py [--ref] [--shapes qkvo,gateup,down,head] [--m 1,2,4,8] [--json out.json]
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

from exllamav2_b200 import ext as ext_c  # noqa: E402
from exllamav2_b200 import synthetic  # noqa: E402
from exllamav2_b200.linear import make_q_matrix  # noqa: E402

DEV = "cuda:0"
SHAPES = {
    "qkvo": dict(K=4096, N=4096, bits=(4,), bits_prop=(1.0,), group_size=128),
    "qkvo54": dict(K=4096, N=4096, bits=(5, 4), bits_prop=(0.1, 0.9), group_size=128),
    "gateup": dict(K=4096, N=11008, bits=(4,), bits_prop=(1.0,), group_size=128),
    "gateup54": dict(K=4096, N=11008, bits=(5, 4), bits_prop=(0.1, 0.9), group_size=128),
    "down": dict(K=11008, N=4096, bits=(4,), bits_prop=(1.0,), group_size=128),
    "down43": dict(K=11008, N=4096, bits=(4, 3), bits_prop=(0.1, 0.9), group_size=128),
    "head": dict(K=4096, N=32000, bits=(6,), bits_prop=(1.0,), group_size=128),
    "tiny_kv": dict(K=2048, N=256, bits=(4,), bits_prop=(1.0,), group_size=128),
    "b3": dict(K=4096, N=4096, bits=(3,), bits_prop=(1.0,), group_size=128),
    "b2": dict(K=4096, N=4096, bits=(2,), bits_prop=(1.0,), group_size=64),
    "b8": dict(K=4096, N=4096, bits=(8,), bits_prop=(1.0,), group_size=128),
    "gptq": dict(K=4096, N=4096, gptq=True),
}


def time_loop(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", action="store_true")
    ap.add_argument("--shapes", default="qkvo,gateup,down,head")
    ap.add_argument("--m", default="1,8")
    ap.add_argument("--total-mb", type=int, default=512)
    ap.add_argument("--json", default=None)
    ap.add_argument("--ctas-per-sm", type=int, default=0)
    ap.add_argument("--phases", action="store_true", help="print per-phase clock stamps of one CTA of the GEMV kernel")
    args = ap.parse_args()
    import ctypes
    ext_c.lib.exl2b_debug_set.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
    if args.ctas_per_sm:
        ext_c.lib.exl2b_debug_set(args.ctas_per_sm, None, 0)
    ref = None
    if args.ref:
        from build_ref import load_ref
        ref = load_ref()
    results = []
    for name in args.shapes.split(","):
        kw = dict(SHAPES[name])
        gptq = kw.pop("gptq", False)
        K, N = kw["K"], kw["N"]
        handles, keep, ref_handles, nbytes = [], [], [], 0
        one = None
        i = 0
        while nbytes < args.total_mb * 2**20:
            w = synthetic.random_gptq(K, N, 128, DEV, seed=i) if gptq else synthetic.random_exl2(device=DEV, seed=i, **kw)
            one = synthetic.algorithmic_bytes(w)
            if ref is not None:
                wr = {k: v.clone() for k, v in w.items()}
                if gptq:
                    none = ext_c.none_tensor
                    hr = ref.make_q_matrix(wr["qweight"], none, none, none, none, none, none, wr["qzeros"], wr["scales"], none, none,
                                           torch.empty((K * N,), dtype=torch.half, device=DEV), K)
                else:
                    wr["q_scale_max"] *= 1 / 256
                    wr["q_perm"], wr["q_invperm"] = wr["q_perm"].short(), wr["q_invperm"].short()
                    wr["q_group_map"] = ref.make_group_map(wr["q_groups"].cpu(), wr["q_weight"].shape[0]).to(DEV)
                    if not keep:
                        tdq = torch.empty((K * N,), dtype=torch.half, device=DEV)
                    hr = ref.make_q_matrix(wr["q_weight"], wr["q_perm"], wr["q_invperm"], wr["q_scale"], wr["q_scale_max"], wr["q_groups"],
                                           wr["q_group_map"], ext_c.none_tensor, ext_c.none_tensor, ext_c.none_tensor, ext_c.none_tensor, tdq, K)
                ref_handles.append(hr)
                keep.append(wr)
            handles.append(make_q_matrix(w))
            keep.append(w)
            nbytes += one
            i += 1
        n = len(handles)
        for M in [int(x) for x in args.m.split(",")]:
            a = torch.randn((M, K), dtype=torch.half, device=DEV)
            c = torch.empty((M, N), dtype=torch.half, device=DEV)
            per_call = synthetic.algorithmic_bytes(keep[-1], M)

            def run_new():
                for h in handles:
                    ext_c.gemm_half_q_half(a, h, c, False)

            if args.phases:
                nl = min(len(handles), 12)
                stamps = torch.zeros((64, 32), dtype=torch.int64, device=DEV)
                for cta in (0, 100):
                    stamps.zero_()
                    stamps[:, 6] = 2**62
                    run_new(); torch.cuda.synchronize()
                    ext_c.lib.exl2b_debug_set(0, stamps.data_ptr(), cta)
                    for h in handles[:nl]:
                        ext_c.gemm_half_q_half(a, h, c, False)
                    torch.cuda.synchronize()
                    ext_c.lib.exl2b_debug_set(0, None, 0)
                    st = stamps.cpu().tolist()
                    t0 = st[0][6]
                    for i in range(nl):
                        r = st[i]
                        print(json.dumps({"shape": name, "M": M, "cta": cta, "launch": i, "grid_start": r[6] - t0, "grid_end": r[7] - t0,
                                          "rel_to_grid_start[start,requested,wait_done,staged,warp0_done,all_warps_done]": [x - r[6] for x in r[:6]], "grid_ns": r[7] - r[6],
                                          "cta[start,prefetched,wait_done,staged,consumed,done]": [x - t0 for x in r[:6]]}), flush=True)
            t_eager = time_loop(run_new, 5)
            # graph-captured cycle (no host launch overhead)
            g = torch.cuda.CUDAGraph()
            stream = torch.cuda.Stream()
            with torch.cuda.stream(stream):
                run_new()
                torch.cuda.synchronize()
                with torch.cuda.graph(g, stream=stream):
                    run_new()
            t_graph = time_loop(g.replay, 10)
            row = dict(shape=name, K=K, N=N, M=M, n_mats=n, bytes_per_call=per_call,
                       new_eager_us=t_eager * 1e3 / n, new_graph_us=t_graph * 1e3 / n,
                       new_eager_gbs=per_call * n / t_eager / 1e6, new_graph_gbs=per_call * n / t_graph / 1e6)
            if ref is not None:
                def run_ref():
                    for h in ref_handles:
                        ref.gemm_half_q_half(a, h, c, True)
                for _ in range(3):          # > 200 calls per shape so the reference's autotuner settles
                    for _ in range(max(1, 260 // n)):
                        run_ref()
                t_ref = time_loop(run_ref, 5)
                row.update(ref_us=t_ref * 1e3 / n, ref_gbs=per_call * n / t_ref / 1e6)
                # the same calls replayed from a CUDA graph: the reference without its host launch overhead
                try:
                    gr = torch.cuda.CUDAGraph()
                    with torch.cuda.stream(stream):
                        run_ref()
                        torch.cuda.synchronize()
                        with torch.cuda.graph(gr, stream=stream):
                            run_ref()
                    t_refg = time_loop(gr.replay, 10)
                    row.update(ref_graph_us=t_refg * 1e3 / n, ref_graph_gbs=per_call * n / t_refg / 1e6)
                except Exception as ex:      # noqa: BLE001
                    row.update(ref_graph_error=str(ex)[:200])
            print(json.dumps(row), flush=True)
            results.append(row)
        for h in handles:
            ext_c.free_q_matrix(h)
        for h in ref_handles:
            ref.free_q_matrix(h)
        del keep, handles
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
