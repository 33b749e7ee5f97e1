"""The batch-1 GEMV's launch plans as gemv_i8_launch builds them (csrc/gemv_i8.cu i8_plan_host, through the host-only hook
exl2b_debug_i8_plan), for tests that replay them (test_i8_smem_operands) or assert which budget branch a launch takes
(test_gpu_full_shapes)."""
import ctypes
import math

import numpy as np

MAX_REGIONS = 6
SMEM_BUDGET = 111 * 1024          # gemv_i8.cu smem_budget: two CTAs co-resident per SM
SMEM_LIMIT = 200 * 1024           # the kernel's attribute and the launch's refusal
ARENA_FLOOR = 2048                # the arena loop stops here even if the CTA still does not fit SMEM_BUDGET


def mat(N, KS, regions, gptq=0):
    """regions: (ks_begin, bits, spg_log2); group_base / off_base derived as qmatrix.cu build_regions does."""
    reg, gbase, off = [], 0, 0
    for i, (ks0, bits, lg) in enumerate(regions):
        ks1 = regions[i + 1][0] if i + 1 < len(regions) else KS
        reg += [ks0, bits, lg, gbase, off]
        gbase += -(-(ks1 - ks0) // (1 << lg))
        off += (ks1 - ks0) * 128 * bits
    rec = [N, KS, gptq, off, len(regions)] + reg
    return rec + [0] * (5 + 5 * MAX_REGIONS - len(rec))


def regions_of(K, plan):
    """The (ks_begin, bits, spg_log2) regions qmatrix.cu build_regions makes of a synthetic checkpoint's groups: EXL2 plans
    (bits, bits_prop, group_size) through synthetic.group_plan, GPTQ ("gptq", group_size, act_order) as one region."""
    from exllamav2_b200 import synthetic
    if plan[0] == "gptq":
        g = plan[1] if plan[1] > 0 else K
        return [(0, 4, int(math.log2(max(32, 1 << math.ceil(math.log2(g))) // 32)))]
    regions, row = [], 0
    groups = synthetic.group_plan(K, list(plan[0]), list(plan[1]), plan[2])
    for i, (bits, rows) in enumerate(groups):
        last_short = i == len(groups) - 1 and i > 0 and groups[i - 1][0] == bits and rows < groups[i - 1][1]
        if not regions or regions[-1][1] != bits or (rows != groups[i - 1][1] and not last_short):
            regions.append((row // 32, bits, int(math.log2(rows // 32))))
        row += rows
    return regions


def plan(mats, ctas, warps=16):
    """(desc, first, busy CTAs, info) of one launch over `mats` (records of mat()); info: arena (bytes per warp), srow (scale-slot
    bytes), smem (dynamic shared memory of a CTA), lcap (longest stage list)."""
    from exllamav2_b200 import ext as ext_c
    f = ext_c.lib.exl2b_debug_i8_plan
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                  ctypes.c_int, ctypes.c_void_p]
    m = np.asarray(sum(mats, []), dtype=np.int32)
    units = sum(-(-r[0] // 32) for r in mats) * mats[0][1]
    cap = units + ctas * warps * 8
    desc = np.zeros((cap, 4), dtype=np.uint32)
    first = np.zeros(ctas * warps + 1, dtype=np.uint32)
    info = np.zeros(6, dtype=np.int32)
    assert f(m.ctypes.data, len(mats), ctas, warps, desc.ctypes.data, cap, first.ctypes.data, len(first), info.ctypes.data) == 0
    C, nd = int(info[0]), int(info[1])
    return desc[:nd], first[: C * warps + 1], C, dict(arena=int(info[2]), srow=int(info[3]), smem=int(info[4]), lcap=int(info[5]))
