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
