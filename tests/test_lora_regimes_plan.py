"""tests/lora_regimes.py's restatement of the LoRA launch geometry (csrc/lora.cu), checked for coverage and against the library's
own bound, and the claim that the GPU case lists of tests/test_gpu_lora_regimes.py reach every branch of the kernel (CPU only)."""
import pytest

import lora_regimes as lr


def test_k_slices_cover_k_once():
    """every K that is a multiple of 32 up to 65536: the cluster's slices are [0, K) in order, each of a multiple of 8 rows but the
    last non-empty one, and empty only past K"""
    for K in range(32, 65536 + 1, 32):
        s = lr.slices(K)
        covered = 0
        for k0, n in s:
            assert k0 == covered or n == 0, (K, s)
            assert n >= 0 and k0 % 8 == 0
            covered += n
        assert covered == K, (K, s)
        assert all(n == lr.kper(K) for _, n in s[:-1] if _ + n < K), (K, s)


def test_slice_regimes():
    assert lr.slices(160)[-1] == (160, 0) and lr.slices(160)[-2] == (144, 16)       # kper 24: an empty and a short slice
    assert lr.slices(96)[-2:] == [(96, 0), (96, 0)]
    assert lr.slices(480)[-1] == (448, 32)
    assert lr.slices(1376)[-1] == (1232, 144)
    assert all(n == 512 for _, n in lr.slices(4096))


@pytest.mark.parametrize("epi,n0,heads", [(lr.ADD, 160, None), (lr.ADD, 8192, None), (lr.ADD, 1376, None),
                                          (lr.ACT_MUL, 480, None), (lr.ACT_MUL, 28672, None), (lr.ACT_MUL, 1376, None),
                                          (lr.QKV, 0, (8, 2, 64)), (lr.QKV, 0, (64, 8, 128)), (lr.QKV, 0, (2, 1, 256)),
                                          (lr.QKV, 0, (4, 2, 80))])
@pytest.mark.parametrize("rows", [1, 8, 17, 40, 129, 1000])
def test_output_units_covered_once(epi, n0, heads, rows):
    """over the grid, every output column of every projection is finished by exactly one thread, and only columns below N"""
    hq, hkv, hd = heads or (0, 0, 0)
    g = lr.launch(epi, 512, rows, n0, hq, hkv, hd)
    owner = [None] * g["units"]
    for x, (u0, u1) in enumerate(g["cta_units"]):
        for u in range(u0, u1):
            assert owner[u] is None
            owner[u] = x
    assert None not in owner
    for sincos, neox in ((hd, True), (hd // 2, True), (hd // 2, False), (hd, False)):
        if epi != lr.QKV and (sincos, neox) != (hd, True):
            continue
        seen = {}
        for u in range(g["units"]):
            for i in range(g["unit_pairs"]):
                c = lr.columns(epi, u, i, n0, hd, hq, hkv, sincos, neox)
                if c is None:
                    continue
                for col in c[:2]:
                    assert col not in seen
                    seen[col] = u
        if epi == lr.QKV:
            want = {(p, c) for p, n in enumerate((hq * hd, hkv * hd, hkv * hd)) for c in range(n)}
        elif epi == lr.ACT_MUL:
            want = {(p, c) for p in (0, 1) for c in range(n0)}
        else:
            want = {(0, c) for c in range(n0)}
        assert set(seen) == want


def test_grid():
    assert lr.launch(lr.QKV, 512, 1, 0, 8, 2, 64)["clusters"] == 2                 # 12 heads
    g = lr.launch(lr.ADD, 512, 129, 512)
    assert g["tiles"] == 17 and g["clusters"] == 1 and g["upc"] == 1               # past one wave: one cluster per row tile
    g = lr.launch(lr.ACT_MUL, 4096, 40, 11008)
    assert g["clusters"] == 3 and g["upc"] == 8


def test_warps_per_group():
    for groups, wpg, idle in ((1, 8, []), (2, 4, []), (3, 2, [6, 7]), (4, 2, []), (5, 1, [5, 6, 7]), (7, 1, [7]), (8, 1, []),
                              (15, 1, []), (64, 1, [])):
        w = lr.warps(8 * groups)
        assert (w["wpg"], w["idle"]) == (wpg, idle)
        taken = sorted(g for gs in w["work"].values() for g in gs)
        assert taken == sorted(list(range(groups)) * wpg)                          # each group by wpg warps
    # wpg > 1: one group per warp, so red[warp] holds one group's partials
    for groups in (1, 2, 3, 4):
        assert all(len(gs) == 1 for gs in lr.warps(8 * groups)["work"].values())


def test_vector_load():
    assert lr.vec_load(16, 8, 24, 0)
    assert not lr.vec_load(16, 8, 24, 2)                                           # A one element off: scalar
    assert not lr.vec_load(12, 8, 0, 0)                                            # 4 columns in the last group
    assert not lr.vec_load(12, 0, 24, 0)                                           # full group, rank 12: scalar
    assert lr.vec_load(8, 0, 1232, 0)


def test_smem_matches_the_library_bound():
    """lora_launch's shared-memory size and its refusal: K = 28672 stages 112 KB at 8 rows; 8 rows of K = 47104 fill the 184 KB
    exactly, and from K = 47105 on the slice rounds up to 5896 rows and is refused"""
    assert lr.smem_bytes(28672, 8) == 114688 and lr.smem_bytes(28672, 3) == 3 * 3584 * 4
    assert lr.smem_bytes(160, 1) == 24 * 4
    assert lr.launch(lr.ADD, 47104, 8, 512)["smem"] == lr.LORA_SMEM_MAX
    for K in (47105, 47168):
        with pytest.raises(ValueError, match="shared memory"):
            lr.launch(lr.ADD, K, 8, 512)
    assert lr.launch(lr.ADD, 47168, 7, 512)["smem"] < lr.LORA_SMEM_MAX             # fewer rows fit
    with pytest.raises(ValueError, match="odd"):
        lr.launch(lr.ADD, 512, 1, 161)


def test_stacked_widths():
    for st in lr.STAGES:
        for R in lr.STACK_WIDTHS:
            ads = lr.stacked(st, R)
            ranks = [r for _, d in ads for p, r in d.items() if p in lr.STAGES[st]]
            assert sum(lr.rank_slots(r) for r in ranks) == R, (st, R)
            assert any(r % 8 for r in ranks) or (R == 512 and st in ("o", "down"))
            assert len(ads) <= 8 and len(ranks) <= lr.LORA_MAX_SEGS
    assert len([1 for _, d in lr.stacked("qkv", 512) for _ in d]) == 24


def test_gpu_cases_reach_every_regime():
    """the launches the GPU case lists make reach every branch named in lora_regimes.REQUIRED"""
    reached = {}
    for name, launches in lr.case_launches().items():
        for l in launches:
            for r in lr.regimes(l):
                reached.setdefault(r, set()).add(name)
    missing = lr.REQUIRED - set(reached)
    assert not missing, f"no GPU case reaches {sorted(missing)}"
    # the regimes that only one list was built for
    assert "tiles_gt_16" in {r for l in lr.case_launches()["long"] for r in lr.regimes(l)}
    assert "slice_gt_100KB" in {r for l in lr.case_launches()["full"] for r in lr.regimes(l)}
    assert "scalar_misaligned" in {r for l in lr.case_launches()["misaligned"] for r in lr.regimes(l)}
    for name in ("empty_slice", "short_slice", "n_tail_add", "n_tail_act_mul", "neox_partial", "gptj_partial"):
        assert "geometry" in reached[name] or name.endswith("partial"), name
    print({k: sorted(v) for k, v in sorted(reached.items())})


def test_constants_match_the_sources():
    """every constant the restatement rests on, read from the constexpr / #define lines of csrc/lora.cu, csrc/lora.cuh and
    include/exl2_b200.h: a change there fails here instead of leaving the plan on stale geometry"""
    import os
    import re
    root = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
    text = ""
    for f in ("exllamav2_b200/csrc/lora.cu", "exllamav2_b200/csrc/lora.cuh", "include/exl2_b200.h"):
        with open(os.path.join(root, f)) as fh:
            text += fh.read()
    defs = {m[0]: m[1] for m in re.findall(r"#define (EXL2B_LORA_\w+) (\d+)", text)}
    consts = {}
    for name, expr in re.findall(r"constexpr int (LORA_\w+) = ([^;]+);", text):
        for k, v in {**defs, **consts}.items():
            expr = re.sub(rf"\b{k}\b", str(v), expr)
        assert re.fullmatch(r"[\d\s*/+()-]+", expr), (name, expr)
        consts[name] = eval(expr)
    want = {n: getattr(lr, n) for n in ("LORA_THREADS", "LORA_WARPS", "LORA_CLUSTER", "LORA_MAX_CTAS", "LORA_SMEM_MAX", "LORA_MT",
                                        "LORA_MAX_RANK", "LORA_MAX_SEGS")}
    assert {n: consts.get(n) for n in want} == want
