"""The wide wgmma launch restated in tests/wide_plan.py, checked on the CPU: tile choice, shared memory, split-K workspace and
buffer sizes, and every restated constant against its constexpr in the source."""
import os
import re

import pytest

import test_gpu_group_structures as gs
import wide_plan as wp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _src(path):
    return open(os.path.join(ROOT, path)).read()


def test_tile_per_row_count():
    assert [wp.tile_for(r) for r in range(1, 65)] == [8] * 8 + [32] * 24 + [64] * 32
    assert all(wp.tile_for(r, chained=False) == 8 for r in range(1, 200))
    with pytest.raises(ValueError, match="64"):
        wp.tile_for(65)


@pytest.mark.parametrize("tw", [32, 64])
@pytest.mark.parametrize("fmt", [f for f, v in gs.FORMATS.items() if v[3]] + ["exl2_54_g128", "gptq_g128_act"])
def test_shared_memory_map(fmt, tw):
    plan = gs.FORMATS[fmt][0] if fmt in gs.FORMATS else {"exl2_54_g128": ((5, 4), (0.1, 0.9), 128),
                                                          "gptq_g128_act": ("gptq", 128, True)}[fmt]
    sb = wp.stage_bytes_of(plan)
    assert sb is not None and 0 < sb <= 4096
    st, total = wp.smem_plan(tw, sb)
    assert 2 <= st <= 4 and total <= wp.TC_SMEM_CAP
    # the combine buffer and fp16 tile overlay the pipeline area, which they must fit
    assert wp.comb_bytes(tw) <= total - wp.header_bytes(tw)
    print(f"{fmt} tw {tw}: stage {sb} B, {st} stages, {total} B")


def test_unstageable_formats_have_no_plan():
    for f, v in gs.FORMATS.items():
        assert (wp.stage_bytes_of(v[0]) is not None) == v[3], f


def test_narrow_map_unchanged():
    """the 8-row kernels keep their header (12 KB) and stage rule"""
    assert wp.header_bytes(8) == 12288
    assert wp.smem_plan(8, 4096) == (2, 12288 + 32768 + 2 * (4096 + 32768))


@pytest.mark.parametrize("preset", list(wp.PRESETS))
def test_workspace_covers_every_launch(preset):
    for name, Ns, K in wp.launches(*wp.PRESETS[preset]):
        for tw in (32, 64):
            need = wp.ws_need(Ns, K, tw)
            assert need <= wp.TC_WIDE_WS_BYTES, (preset, name, tw, need)
        assert wp.ws_need(Ns, K, 8) <= wp.TC_WS_BYTES
        assert max(Ns) * 0 + K * 64 * 2 * 3 <= wp.TC_WIDE_XP_BYTES


def test_buffer_sizes():
    assert wp.chain_buffer_bytes(4096, 8) == (4096 * 16, 34 * 8 * 4)
    assert wp.chain_buffer_bytes(4096, 9) == (4096 * 128, 34 * 64 * 4)
    assert wp.TC_WIDE_XP_BYTES == 3 * 65536 * 64 * 2


PINS = [
    ("exllamav2_b200/csrc/gemv.cuh", r"constexpr int GEMV_MTOK = (\d+);", wp.GEMV_MTOK),
    ("exllamav2_b200/csrc/gemv.cuh", r"constexpr int GEMV_MAX_CHAIN_ROWS = (\d+);", wp.GEMV_MAX_CHAIN_ROWS),
    ("exllamav2_b200/csrc/gemv.cuh", r"TC_WS_BYTES = \(size_t\)(\d+) << 20;", wp.TC_WS_BYTES >> 20),
    ("exllamav2_b200/csrc/gemv.cuh", r"TC_WIDE_WS_BYTES = \(size_t\)(\d+) << 20;", wp.TC_WIDE_WS_BYTES >> 20),
    ("exllamav2_b200/csrc/gemv.cuh", r"TC_WIDE_XP_BYTES = \(size_t\)GEMV_MAX_MATS \* 65536 \* (\d+);", 128),
    ("exllamav2_b200/csrc/gemm_tc.cu", r"constexpr int TC_MAX_STAGES = (\d+);", wp.TC_MAX_STAGES),
    ("exllamav2_b200/csrc/gemm_tc.cu", r"constexpr int TC_SMEM_CAP = (\d+) \* 1024;", wp.TC_SMEM_CAP // 1024),
    ("exllamav2_b200/csrc/gemm_tc.cu", r"const long long F = (\d+);", wp.SPLIT_F),
    ("exllamav2_b200/csrc/qmatrix.cu", r"const size_t slots = wide \? (\d+) : 8;", 64),
]
FORMULAS = [
    ("exllamav2_b200/csrc/gemm_tc.cu", "constexpr int tc_act_stage(int tw) { return 128 * tw * 2; }", wp.act_stage),
    ("exllamav2_b200/csrc/gemm_tc.cu", "constexpr int tc_misc_bytes(int tw) { return tw > GEMV_MTOK ? 128 + 4 * tw : 128; }", wp.misc_bytes),
    ("exllamav2_b200/csrc/gemm_tc.cu", "constexpr int tc_ssq_bytes(int tw) { return 4 * tw * 4; }", wp.ssq_bytes),
    ("exllamav2_b200/csrc/gemm_tc.cu", "constexpr int tc_corr_floats(int tw) { return 2 * 2 * 4 * 2 * tw; }", wp.corr_floats),
    ("exllamav2_b200/csrc/gemm_tc.cu", "constexpr int tc_red_floats(int tw) { return tw * 128; }", wp.red_floats),
    ("exllamav2_b200/csrc/gemm_tc.cu", "constexpr int tc_comb_bytes(int tw) { return 2 * tw * 128 * 4 + tw * 128 * 2; }", wp.comb_bytes),
    ("exllamav2_b200/csrc/gemv.cuh", "constexpr int tc_tile(int rows) { return rows <= GEMV_MTOK ? GEMV_MTOK : rows <= 32 ? 32 : 64; }", wp.tile_for),
]


@pytest.mark.parametrize("path,pat,want", PINS, ids=[p[1][:40] for p in PINS])
def test_constants_pinned(path, pat, want):
    m = re.search(pat, _src(path))
    assert m and int(m.group(1)) == want


@pytest.mark.parametrize("path,line,fn", FORMULAS, ids=[f[1][14:40] for f in FORMULAS])
def test_formulas_pinned(path, line, fn):
    """the source line is the restatement's formula: evaluated as Python over every tile width it takes"""
    assert line in _src(path)
    body = line.split("return ", 1)[1].rsplit(";", 1)[0]
    body = re.sub(r"(\w+) > (\w+) \? (.+?) : (.+)$", r"(\3) if \1 > \2 else (\4)", body)
    body = re.sub(r"rows <= GEMV_MTOK \? GEMV_MTOK : rows <= 32 \? 32 : 64", "8 if rows <= 8 else (32 if rows <= 32 else 64)", body)
    arg = "rows" if "rows" in line else "tw"
    for v in ((1, 8, 9, 31, 32, 33, 64) if arg == "rows" else (8, 32, 64)):
        assert eval(body, {"GEMV_MTOK": 8, arg: v}) == fn(v), (line, v)
    assert "tc_header_bytes" in _src("exllamav2_b200/csrc/gemm_tc.cu")


# ---- the per-CTA walk (wide_plan.walk) at full model size ----------------------------------------------------------------------

def _preset_plans():
    """(name, launches [(name, [(N, plan)], K, paired)]) of every shipped preset's plans, every MLP plan it cycles through,
    plus the 8-bit g128 plan of the exl2-8bpw test model"""
    from exllamav2_b200.model import PRESETS
    out = []
    for name, mk in PRESETS.items():
        c = mk()
        hid, inter, H, KVH, hd, p = c.hidden_size, c.intermediate_size, c.num_heads, c.num_kv_heads, c.head_dim, c.plan
        ls = [("qkv", [(H * hd, p.attn), (KVH * hd, p.attn), (KVH * hd, p.attn)], hid, False), ("o", [(hid, p.attn)], H * hd, False),
              ("head", [(c.vocab_size, p.head)], hid, False)]
        for i, mp in enumerate(p.mlp):
            ls += [(f"gate_up{i}", [(inter, mp), (inter, mp)], hid, True), (f"down{i}", [(hid, mp)], inter, False)]
        out.append((name, ls))
    out.append(("exl2-8bpw", [("all", [(512, wp.HEAD8)], 512, False)]))
    return out


def _shape_launches(preset):
    """wp.PRESETS' shapes in plans of their size class: 7B in the 4.0 bpw mix, 70B in 2.5 bpw, the rest 4-bit / 6-bit g128"""
    hid, inter, H, KVH, hd, vocab = wp.PRESETS[preset]
    a, m = {"7B": (wp.M54, wp.M43), "70B": (wp.A70, wp.M70)}.get(preset, (((4,), (1.0,), 128),) * 2)
    return [("qkv", [(H * hd, a), (KVH * hd, a), (KVH * hd, a)], hid, False), ("o", [(hid, a)], H * hd, False),
            ("gate_up", [(inter, m), (inter, m)], hid, True), ("down", [(hid, m)], inter, False),
            ("head", [(vocab, wp.HEAD6)], hid, False)]


WALK_CASES = [(f"{p}-{n}", Ns, K, pr) for p in wp.PRESETS for n, Ns, K, pr in _shape_launches(p)] + \
             [(f"{b}-{n}", Ns, K, pr) for b in wp.FULL_BLOCKS for n, Ns, K, pr in wp.block_launches(b)]


def test_cta_of_unit_is_the_owner():
    """tc_cta_of_unit inverts the unit ranges [b U / G, (b + 1) U / G), for grids that divide U and grids that do not"""
    for U, G in ((128 * 250, 132), (448 * 128, 132), (86 * 344, 128), (1188 * 256, 132), (7, 7), (1000, 3)):
        owner = [b for b in range(G) for _ in range(b * U // G, (b + 1) * U // G)]
        assert owner == [wp.cta_of_unit(x, G, U) for x in range(U)], (U, G)


@pytest.mark.parametrize("tw", [32, 64])
@pytest.mark.parametrize("case", WALK_CASES, ids=[c[0] for c in WALK_CASES])
def test_walk_tiles_and_hands_off(case, tw):
    """Per launch, as every CTA of the wide kernel walks it:
      * the raw segments cover every unit once, and the snapped ranges of all CTAs and both warpgroups cover each strip's
        slabs exactly once, each range starting and ending on a group start;
      * a contributor's slot jc is below maxc (its partials stay inside its strip's workspace), and the slots a strip's
        contributors write are exactly 0 .. nc - 1, the ones the finisher sums;
      * every counter is reached by exactly `expected` arrivals, the count each arriving CTA computes -- for gate|up, gate's and
        up's contributors together."""
    name, Ns, K, paired = case
    from i8_plans import regions_of
    G, maxc, aligned, segs = wp.launch_walk(Ns, K, paired, tw)
    KS = K // 32
    units = {}
    for s in segs:
        key = (s["mat"], s["strip"])
        units.setdefault(key, []).append(s["ks"])
    assert sorted(units) == [(m, st) for m, (n, _) in enumerate(Ns) for st in range(-(-n // 128))]
    for (m, st), rs in units.items():
        assert sorted(rs)[0][0] == 0 and all(a[1] == b[0] for a, b in zip(sorted(rs), sorted(rs)[1:])) and max(rs)[1] == KS
        regions = regions_of(K, Ns[m][1])
        snapped = sorted(r for s in segs if (s["mat"], s["strip"]) == (m, st) for r in s["wg"] if r[0] < r[1])
        assert snapped[0][0] == 0 and snapped[-1][1] == KS, (name, m, st)
        assert all(a[1] == b[0] for a, b in zip(snapped, snapped[1:])), (name, m, st, snapped)
        assert all(wp.group_start(regions, KS, e) == e for r in snapped for e in r), (name, m, st)
    slots, arrivals = {}, {}
    for s in segs:
        if s["alone"]:
            assert s["nc"] == 1 and s["jc"] == 0
            continue
        assert 0 <= s["jc"] < maxc, (name, s)
        slots.setdefault(s["slot"], []).append(s["jc"])
        arrivals.setdefault(s["counter"], []).append(s["expected"])
    for slot, js in slots.items():
        nc = [s["nc"] for s in segs if s["slot"] == slot]
        assert sorted(js) == list(range(nc[0])) and len(set(nc)) == 1, (name, slot, js)
    for cidx, exp in arrivals.items():
        assert len(set(exp)) == 1 and exp[0] == len(exp), (name, cidx, exp)
        if paired:   # gate's and up's writers of that strip
            st = cidx
            assert exp[0] == len(slots[st]) + len(slots[sum(-(-n // 128) for n, _ in Ns[:1]) + st]), (name, cidx)
    assert 2 <= maxc and len(slots) * maxc * wp.red_floats(tw) * 4 <= wp.TC_WIDE_WS_BYTES


def _full_regimes():
    out = {}
    for b in wp.FULL_BLOCKS:
        for n, Ns, K, paired in wp.block_launches(b):
            G, maxc, aligned, segs = wp.launch_walk(Ns, K, paired)
            out[(b, n)] = dict(wp.regimes(segs, G), grid=G, aligned=aligned,
                               stages={tw: wp.smem_plan(tw, max(wp.stage_bytes_of(p) for _, p in Ns))[0] for tw in (32, 64)},
                               paired_spread=paired and max(len({s["strip"] for s in segs if s["cta"] == c}) for c in range(G)) > 1)
    return out


def test_full_cases_reach_every_regime():
    """The launches of test_gpu_wide_full_shapes.py reach every stream-K regime of the wide kernels: 2, 3, 5 and 9 segments
    in one CTA, CTAs that cross from q to k and k to v, empty snapped segments, empty warpgroups, the paired gate|up finisher
    with contributors that own other strips, and both halves of the grid rule -- and the smaller shapes of the other wide tests
    reach none of it."""
    r = _full_regimes()
    for k, v in sorted(r.items()):
        print(k, v)
    assert {v["max_segs"] for v in r.values()} >= {1, 2, 3, 5, 9}
    assert r[("7b-4.0bpw", "qkv")]["max_segs"] == 2 and r[("7b-4.0bpw", "qkv")]["grid"] == 132
    for k in (("7b-4.0bpw", "gate_up0"), ("7b-4.0bpw", "head32000_6")):
        assert (r[k]["grid"], r[k]["max_segs"], r[k]["empty_segs"], r[k]["empty_wg"]) == (132, 3, 4, 8), k
    assert r[("70b-2.5bpw", "qkv")]["crossings"] == 2 and r[("70b-2.5bpw", "qkv")]["max_segs"] == 2
    assert r[("70b-2.5bpw", "gate_up0")]["max_segs"] == 5
    assert r[("70b-2.5bpw", "head152064_6")]["max_segs"] == 9
    assert any(v["paired_spread"] for v in r.values())
    assert {v["aligned"] for v in r.values()} == {True, False}
    # the small shapes: one segment per CTA, aligned split, nothing else
    small = [(512, 1408, 8, 8, 64, 512), (256, 704, 4, 2, 64, 512), (1024, 2816, 8, 4, 128, 1024), (1536, 4096, 28, 4, 128, 2048)]
    for hid, inter, H, KVH, hd, vocab in small:
        for n, Ns, K in wp.launches(hid, inter, H, KVH, hd, vocab):
            G, _, aligned, segs = wp.launch_walk([(N, wp.M54) for N in Ns], K, n == "gate_up")
            assert G <= 132 and wp.regimes(segs, G) == dict(max_segs=1, crossings=0, empty_segs=0, empty_wg=0), (hid, n)


def test_full_cases_reach_every_stage_count():
    """every (TW, stage count) pair the presets' launches produce is among the full-size cases'"""
    assert [wp.smem_plan(tw, wp.stage_bytes_of(p))[0] for p in (wp.M54, wp.HEAD6, wp.HEAD8) for tw in (32, 64)] == [4, 3, 4, 2, 3, 2]
    want = {(tw, wp.smem_plan(tw, max(wp.stage_bytes_of(p) for _, p in Ns))[0])
            for _, ls in _preset_plans() for _, Ns, _, _ in ls if all(wp.stage_bytes_of(p) for _, p in Ns) for tw in (32, 64)}
    got = {(tw, st) for v in _full_regimes().values() for tw, st in v["stages"].items()}
    print("presets", sorted(want), "full cases", sorted(got))
    assert want <= got


WALK_LINES = [     # the kernel's walk and hand-off, as wide_plan.walk / grid_rule restate them
    "const int u0 = (int)((unsigned)blockIdx.x * U / G), u1 = (int)(((unsigned)blockIdx.x + 1u) * U / G);",
    "while (mi + 1 < P.num_mats && u >= P.mat[mi + 1].unit_begin) ++mi;",
    "const int strip = local / KS, ks_a = local - strip * KS;",
    "const int seg = min(KS - ks_a, u1 - u);",
    "const int ks0 = tc_group_start(w, ks_a), ks1 = tc_group_start(w, ks_a + seg);",
    "const int ksm = tc_group_start(w, ks0 + ((ks1 - ks0 + 1) >> 1));",
    "const int my0 = wg ? ksm : ks0, my1 = wg ? ks1 : ksm;",
    "return R.ks_begin + (((ks - R.ks_begin) >> R.spg_log2) << R.spg_log2);",
    "if (ks >= w.KS) return w.KS;",
    "return (int)(((x + 1u) * G - 1u) / U);",
    "const int first_cta = tc_cta_of_unit(sb, G, U), last_cta = tc_cta_of_unit(sb + KS - 1, G, U);",
    "const int nc = last_cta - first_cta + 1, jc = (int)blockIdx.x - first_cta;",
    "const bool alone = nc == 1 && !paired;",
    "float* wsp = P.ws + ((size_t)gs * P.maxc + jc) * RED;",
    "expected += tc_cta_of_unit(ob + KS - 1, G, U) - tc_cta_of_unit(ob, G, U) + 1;",
    "cidx = P.mat[0].strip_begin + strip;",
    "u += seg;",
    "const int S = (int)std::min<long long>(slots / strips, std::max(1, P.KS / 8));",
    "const long long cost_aligned = F + (P.KS + S - 1) / S;",
    "const long long cost_stream = ((L + P.KS - 1) / P.KS + 1) * F + L;",
    "if (cost_aligned <= cost_stream) grid_ll = (long long)strips * S;",
    "P.maxc = (int)(((long long)P.KS * grid) / units) + 2;",
    "const int ctas_per_sm = wide ? 1 : g_tc_ctas_per_sm;",
]


@pytest.mark.parametrize("line", WALK_LINES, ids=[l[:40] for l in WALK_LINES])
def test_walk_lines_pinned(line):
    assert line in _src("exllamav2_b200/csrc/gemm_tc.cu")
