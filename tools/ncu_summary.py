"""Summarise an .ncu-rep (one kernel, --set full --import-source on) as markdown: python tools/ncu_summary.py rep.ncu-rep > out.md
Runs on the CPU box (ncu -i ... --page raw/source --csv)."""
import csv, io, subprocess, sys
from collections import Counter

rep = sys.argv[1]
def page(p):
    out = subprocess.run(["ncu", "-i", rep, "--page", p, "--csv"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True).stdout
    return list(csv.reader(io.StringIO(out)))
raw = page("raw")
hdr, units, vals = raw[0], raw[1], raw[2]
m = {h: (v, u) for h, u, v in zip(hdr, units, vals)}
def g(k):
    v, u = m.get(k, ("n/a", ""))
    return f"{v} {u}".strip()
print(f"# ncu summary: {m.get('Kernel Name', ('?',''))[0]}\n")
print(f"source: `{rep}` (ncu --set full --clock-control none --import-source on; cold-cache, serialised replay -- shares, not absolutes)\n")
print("| metric | value |\n|---|---|")
for k in ["gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic",
          "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "sm__warps_active.avg.pct_of_peak_sustained_active",
          "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct",
          "sm__inst_executed.sum.per_cycle_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
          "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "sm__cycles_active.avg"]:
    print(f"| `{k}` | {g(k)} |")
print("\n## warp stall reasons (warps stalled per issue-active cycle)\n\n| reason | ratio |\n|---|---|")
st = [(h.replace("smsp__average_warps_issue_stalled_", "").replace("_per_issue_active.ratio", ""), float(v)) for h, v in zip(hdr, vals)
      if h.startswith("smsp__average_warps_issue_stalled_") and h.endswith("_per_issue_active.ratio")]
for n, v in sorted(st, key=lambda t: -t[1]):
    print(f"| {n} | {v:.2f} |")
src = page("source")
if len(src) > 2:
    h2, data = src[1], src[2:]
    iS, iN, iE = h2.index("Source"), h2.index("# Samples"), h2.index("Instructions Executed")
    tot = sum(int(r[iE]) for r in data); totS = max(1, sum(int(r[iN]) for r in data))
    op, ops = Counter(), Counter()
    for r in data:
        t = r[iS].strip().split()
        o = (t[1] if t[0].startswith("@") else t[0]).split(".")[0]
        op[o] += int(r[iE]); ops[o] += int(r[iN])
    print(f"\n## SASS mix ({tot} warp instructions, {totS} stall samples)\n\n| opcode | executed | share | stall samples |\n|---|---|---|---|")
    for o, c in op.most_common(18):
        print(f"| {o} | {c} | {100*c/tot:.1f}% | {100*ops[o]/totS:.1f}% |")
    present = [k for k in ("HGMMA", "UBLKCP", "SYNCS", "WARPSYNC") if any(k in r[iS] for r in data)]
    print(f"\nwgmma / TMA mnemonics present in the SASS: {', '.join(present)}")
