"""Host-side checks of where the batch-1 GEMV's main loop gets its operands (no GPU needed).

gemv_i8_kernel reads a group's scale row and its stage descriptors from shared memory:
  * a flush stage brings its group's 32-column scale row into slot s % 8 of the warp's scale ring, on stage s's mbarrier;
  * descriptors 0..7 are loaded before the first request, and stage s brings descriptor s + 8 into slot (s + 8) % 16 of the
    warp's list window, on the same mbarrier.
Here the kernel's request / wait / consume order is replayed over the plans gemv_i8_launch builds (exl2b_debug_i8_plan) for the
flagship 7B launch structures and the GPTQ and 70B presets: every read must find the entry it expects, delivered by a barrier
that has already been waited for, and the CTA must fit the 111 KB that keeps two CTAs co-resident per SM."""
import numpy as np
import pytest

from i8_plans import SMEM_BUDGET, SMEM_LIMIT, ARENA_FLOOR, mat as _mat, plan as _plan_on

I8_BARS, I8_LWIN = 8, 16
SMS, WARPS = 132, 16


def _plan(mats, ctas=SMS, warps=WARPS):
    return _plan_on(mats, ctas, warps)


K4, K11, K8, K28, K64 = 128, 344, 256, 896, 2048    # slabs (32 rows) of K = 4096, 11008, 8192, 28672, 65536
M54_4K = [(0, 5, 2), (13, 4, 2)]
M54_11K = [(0, 5, 2), (36, 4, 2)]
M43_4K = [(0, 4, 2), (13, 3, 2)]
STRUCTURES = {
    # llama2-7b-4.0bpw, the decode benchmark's launches
    "7b q|k|v": [_mat(4096, K4, M54_4K)] * 3,
    "7b o": [_mat(4096, K4, M54_4K)],
    "7b gate|up [5,4]": [_mat(11008, K4, M54_4K)] * 2,
    "7b gate|up [4,3]": [_mat(11008, K4, M43_4K)] * 2,
    "7b down": [_mat(4096, K11, M54_11K)],
    "7b head": [_mat(32000, K4, [(0, 6, 2)])],
    # llama2-7b-gptq-g128-act: 128-byte scale | zero rows
    "gptq q|k|v": [_mat(4096, K4, [(0, 4, 2)], gptq=1)] * 3,
    "gptq gate|up": [_mat(11008, K4, [(0, 4, 2)], gptq=1)] * 2,
    "gptq down": [_mat(4096, K11, [(0, 4, 2)], gptq=1)],
    # llama2-70b-2.5bpw: g64 MLP (every second slab flushes), the longest stage lists
    # (attention [4,3] at 0.1 / 0.9, g128: ceil(819.2 / 128) = 7 groups of 4 bits, 28 slabs)
    "70b q|k|v": [_mat(8192, K8, [(0, 4, 2), (28, 3, 2)]), _mat(1024, K8, [(0, 4, 2), (28, 3, 2)]), _mat(1024, K8, [(0, 4, 2), (28, 3, 2)])],
    "70b o": [_mat(8192, K8, [(0, 4, 2), (28, 3, 2)])],
    "70b head": [_mat(32000, K8, [(0, 6, 2)])],
    "70b gate|up": [_mat(28672, K8, [(0, 3, 1), (78, 2, 1)])] * 2,
    "70b down": [_mat(8192, K28, [(0, 3, 1), (270, 2, 1)])],
    # small cases of the GPU tests: every stage flushes (8-bit g32), groups spanning stages (g256), ragged N
    "8-bit g32 + 2-bit g64": [_mat(512, 64, [(0, 8, 0), (5, 2, 1)])],
    "g256": [_mat(1024, 64, [(0, 4, 3)])],
    "N = 1000": [_mat(1000, 16, [(0, 3, 0), (3, 2, 2)])],
    "K = 16384 8-bit g32": [_mat(4096, 512, [(0, 8, 0)])],
    # over the budget (test_gpu_full_shapes runs both): the staged row alone is KS * 64 B, so the arenas shrink to the floor and the
    # CTA still needs more than 111 KB -- it runs one CTA per SM
    "70b gptq down": [_mat(8192, K28, [(0, 4, 2)], gptq=1)],
    "K = 65536 4-bit g128": [_mat(1024, K64, [(0, 4, 2)])],
}
OVER_BUDGET = {"70b gptq down", "K = 65536 4-bit g128"}


def _replay(lst, n_pre):
    """The kernel's order of events for one warp; returns (window refills, stages that refilled a slot read later)."""
    nst = len(lst)
    window = {}                 # slot -> (descriptor index, carrier stage or -1 for the up-front load)
    scales = {}                 # slot -> flush stage whose scale row it holds
    waited = -1                 # highest stage whose barrier has been waited for
    refills = 0

    def read_desc(i):
        slot = i % I8_LWIN
        assert slot in window and window[slot][0] == i, f"descriptor {i} overwritten or never delivered"
        assert window[slot][1] <= waited, f"descriptor {i} read before its barrier (stage {window[slot][1]}) was waited for"

    def issue(t):
        nonlocal refills
        flags = int(lst[t][2] >> 18) & 15
        if flags & 1:
            prev = scales.get(t % I8_BARS)
            assert prev is None or prev < t and prev <= waited, f"scale slot of stage {t} still holds unread stage {prev}"
            scales[t % I8_BARS] = t
        if t + I8_BARS < nst:
            slot = (t + I8_BARS) % I8_LWIN
            if slot in window:
                assert window[slot][0] <= waited, f"window slot of descriptor {window[slot][0]} reused before it was consumed"
            window[slot] = (t + I8_BARS, t)
            refills += 1

    for i in range(min(I8_BARS, nst)):
        window[i] = (i, -1)
    assert n_pre <= I8_BARS
    for t in range(n_pre):
        read_desc(t)
        issue(t)
    next_req = n_pre
    for s in range(nst):
        read_desc(s)
        nreq = int(lst[s][3] >> 24) & 15
        assert s < next_req, "stage waited for before it was requested"
        waited = s
        for j in range(nreq):
            read_desc(next_req + j)
        if (int(lst[s][2] >> 18) & 15) & 1:
            assert scales.get(s % I8_BARS) == s, f"scale row of stage {s} overwritten or never requested"
        for j in range(nreq):
            issue(next_req + j)
        next_req += nreq
        assert next_req - (s + 1) <= I8_BARS
    assert next_req == nst
    return refills


@pytest.mark.parametrize("name", list(STRUCTURES))
def test_smem_operands(name):
    mats = STRUCTURES[name]
    desc, first, C, info = _plan(mats)
    if name in OVER_BUDGET:
        assert info["arena"] == ARENA_FLOOR and SMEM_BUDGET < info["smem"] <= SMEM_LIMIT, info
    else:
        assert info["smem"] <= SMEM_BUDGET, f"{info['smem']} B of dynamic shared memory"
    assert info["srow"] == (128 if any(m[2] for m in mats) else 64)
    assert info["arena"] >= ARENA_FLOOR
    n_pre = (first >> 26).astype(int)
    first = (first & 0x3FFFFFF).astype(np.int64)
    longest = 0
    for cw in range(C * WARPS):
        lst = desc[first[cw]: first[cw + 1]]
        refills = _replay(lst, int(n_pre[cw]))
        assert refills == max(0, len(lst) - I8_BARS), "every descriptor past the first 8 arrives with the stage 8 before it"
        longest = max(longest, len(lst))
    assert longest == info["lcap"]


@pytest.mark.parametrize("name", ["70b gate|up", "K = 16384 8-bit g32"])
def test_long_lists_refill_the_window(name):
    # lists longer than the window: their later descriptors can only come from refills (test_smem_operands replays them)
    _, first, _, info = _plan(STRUCTURES[name])
    assert info["lcap"] >= 2 * I8_LWIN
    first = (first & 0x3FFFFFF).astype(np.int64)
    assert max(np.diff(first)) == info["lcap"]


def test_gptq_rows_need_the_wider_slot():
    # 32 columns of scale | zero << 16 are 128 bytes; a launch without GPTQ matrices keeps 64-byte slots and a larger arena
    _, _, _, exl2 = _plan([_mat(4096, K4, [(0, 4, 2)])])
    _, _, _, gptq = _plan([_mat(4096, K4, [(0, 4, 2)], gptq=1)])
    assert (exl2["srow"], gptq["srow"]) == (64, 128)
    assert exl2["arena"] >= gptq["arena"] and exl2["smem"] <= SMEM_BUDGET and gptq["smem"] <= SMEM_BUDGET
