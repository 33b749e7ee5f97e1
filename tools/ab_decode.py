"""A/B of the decode benchmark between two source trees on the same GPU.

    python tools/ab_decode.py BASE_TREE NEW_TREE [--runs 5] [--out DIR] [-- extra bench.py arguments]

Runs `bench.py --no-ref-ext --no-cpu --dump-outputs ...` from each tree alternately (base, new, base, new, ...), each in a
fresh process, and prints the median / min / max of `value` (tok/s) and `roofline.achieved` (GB/s) per tree, whether the
dumped logits and next token of every run are byte-identical to the base tree's first run, and the card and power limit
(read-only `nvidia-smi --query-gpu`).  Each tree must already be built (`python -m exllamav2_b200.build` inside it).
The last line is one JSON object with all of it; with --out the per-run JSON lines and dumps are kept there."""
from __future__ import annotations

import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile


def card() -> str:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0] if r.stdout.strip() else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def run_bench(tree: str, dump: str, extra: list[str]) -> dict:
    cmd = [sys.executable, "bench.py", "--gpus", "1", "--no-ref-ext", "--no-cpu", "--dump-outputs", dump, *extra]
    env = {k: v for k, v in os.environ.items() if k != "PYTHONPATH"}
    r = subprocess.run(cmd, cwd=tree, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{") and '"metric"' in ln]
    if r.returncode != 0 or not lines:
        sys.stderr.write(r.stdout[-4000:])
        raise RuntimeError(f"bench.py failed in {tree} (exit {r.returncode})")
    return json.loads(lines[-1])


def same_bytes(a: str, b: str) -> bool:
    names = sorted(f for f in os.listdir(a) if f.endswith(".npy"))
    if not names or names != sorted(f for f in os.listdir(b) if f.endswith(".npy")):
        return False
    for n in names:
        with open(os.path.join(a, n), "rb") as fa, open(os.path.join(b, n), "rb") as fb:
            if fa.read() != fb.read():
                return False
    return True


def spread(xs: list[float]) -> dict:
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "runs": xs}


def main() -> None:
    argv = sys.argv[1:]
    extra = []
    if "--" in argv:
        i = argv.index("--")
        argv, extra = argv[:i], argv[i + 1:]
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("base")
    ap.add_argument("new")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default=None, help="keep per-run JSON lines and output dumps here")
    args = ap.parse_args(argv)
    trees = {"base": os.path.abspath(args.base), "new": os.path.abspath(args.new)}
    out = os.path.abspath(args.out) if args.out else tempfile.mkdtemp(prefix="ab_decode_")
    os.makedirs(out, exist_ok=True)
    gpu = card()
    print(f"card: {gpu}", flush=True)
    res = {k: [] for k in trees}
    identical = {k: [] for k in trees}
    for i in range(args.runs):
        for k, tree in trees.items():
            dump = os.path.join(out, f"{k}_{i}")
            shutil.rmtree(dump, ignore_errors=True)
            line = run_bench(tree, dump, extra)
            res[k].append(line)
            with open(os.path.join(out, "runs.jsonl"), "a") as f:
                f.write(json.dumps({"tree": k, "run": i, **line}) + "\n")
            identical[k].append(same_bytes(os.path.join(out, "base_0"), dump))
            print(f"{k:4s} run {i}: {line['value']:8.2f} tok/s  roofline {line['roofline']['achieved']:8.1f} GB/s  "
                  f"launches/step {line['launches_per_step']}  outputs == base_0: {identical[k][-1]}", flush=True)
    summary = {"card": gpu, "bench_args": extra, "out": out}
    for k in trees:
        summary[k] = {"tree": trees[k], "value": spread([r["value"] for r in res[k]]),
                      "roofline_achieved": spread([r["roofline"]["achieved"] for r in res[k]]),
                      "launches_per_step": sorted({r["launches_per_step"] for r in res[k]}),
                      "outputs_identical_to_base": all(identical[k])}
    vb, vn = summary["base"]["value"], summary["new"]["value"]
    summary["median_gain"] = vn["median"] / vb["median"] - 1.0
    summary["new_slowest_beats_base_fastest"] = vn["min"] > vb["max"]
    for k in trees:
        v, a = summary[k]["value"], summary[k]["roofline_achieved"]
        print(f"{k:4s} tok/s median {v['median']:8.2f} [{v['min']:.2f}, {v['max']:.2f}]   roofline GB/s median {a['median']:8.1f} "
              f"[{a['min']:.1f}, {a['max']:.1f}]   outputs identical: {summary[k]['outputs_identical_to_base']}")
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
