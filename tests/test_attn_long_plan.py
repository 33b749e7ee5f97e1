"""tests/attn_long_plan.py's restatement of the long-context decode regime (csrc/attn_q4.cu attn_launch_plan, pass_len,
attn_q4_passes_kernel), pinned to the figures DESIGN.md §3.4 states (CPU only)."""
import numpy as np
import pytest

import attn_long_plan as lp
import attn_regimes as ar

FMTS = [(w, hd) for w in (4, 6, 8) for hd in (64, 128)]
SHAPES = [(32, 1), (32, 4), (32, 8), (32, 9), (64, 1), (64, 4), (28, 10), (8, 1)]


@pytest.mark.parametrize("wbits,hd", FMTS)
@pytest.mark.parametrize("H,B", SHAPES)
def test_regime_taken_exactly_where_todays_plan_does_not_fit(wbits, hd, H, B):
    """Passes only for q_len 1, and exactly where attn_regimes.smem_bytes says the single-pass plan exceeds 200 KB; a launch
    that fits keeps its plan.  q_len 2-8 never takes the regime (their refusal stays)."""
    edge = lp.largest_fit(wbits, hd, H, B)
    for ctx in (4096, edge - ar.PAGE, edge, edge + ar.PAGE, 2 * edge, 131072):
        for q_len in (1, 2, 8):
            nsplit = ar.nsplit_of(q_len, ctx, H, B)
            fits = ar.smem_bytes(wbits, hd, q_len, ctx, nsplit)["fits"]
            p = lp.long_plan(wbits, hd, H, B, q_len, ctx)
            assert p["nsplit"] == nsplit
            assert p["passes"] == (q_len == 1 and not fits)
            if not p["passes"]:
                assert p["pass_len"] == 0 and p["smem"] == ar.smem_bytes(wbits, hd, q_len, ctx, nsplit)["smem"]
            assert p["passes"] == (q_len == 1 and ctx > edge)


# pass_len and the launch's shared memory at a 131072-position cache (512 pages, 32 heads, B = 9), and the largest page table accepted
PINNED = {  # (wbits, hd): (pass_len, smem at 512 pages, most pages accepted)
    (4, 64): (17408, 115792, 39660), (4, 128): (6400, 115808, 28648),
    (6, 64): (18944, 116048, 41132), (6, 128): (9472, 116320, 31592),
    (8, 64): (17920, 116304, 40044), (8, 128): (7168, 115808, 29416),
}


@pytest.mark.parametrize("wbits,hd", FMTS)
def test_pass_len_and_footprint(wbits, hd):
    """The pass fills what the page table and the fixed map leave of the 114 KB target, in multiples of 256 positions; the CTA then fits
    beside a 111 KB GEMV CTA on one SM (228 KB, 1 KB reserved per CTA)."""
    pass_len, smem, _ = PINNED[(wbits, hd)]
    p = lp.long_plan(wbits, hd, 32, 9, 1, 131072)
    assert p["passes"] and p["pass_len"] == pass_len and p["smem"] == smem
    assert p["smem"] <= lp.PASS_SMEM < p["smem"] + lp.PASS_ALIGN * 4
    assert p["smem"] + 16 + 1024 + 111 * 1024 + 1024 <= 228 * 1024
    assert pass_len % lp.PASS_ALIGN == 0 and pass_len >= p["stage"] and pass_len % p["sub"] == 0
    # the pass length follows the page table: longer caches leave less room
    a = lp.long_plan(wbits, hd, 32, 9, 1, 65536)["pass_len"]
    b = lp.long_plan(wbits, hd, 32, 9, 1, 1 << 20)["pass_len"]
    assert a >= pass_len >= b >= lp.PASS_MIN


@pytest.mark.parametrize("wbits,hd", FMTS)
def test_largest_page_table_and_one_more(wbits, hd):
    """Refused only when the page table plus a pass of PASS_MIN positions exceeds 200 KB."""
    most = PINNED[(wbits, hd)][2]
    assert lp.largest_page_table(wbits, hd) == most
    ok = lp.long_plan(wbits, hd, 8, 1, 1, most * ar.PAGE)
    bad = lp.long_plan(wbits, hd, 8, 1, 1, (most + 1) * ar.PAGE)
    assert ok["passes"] and ok["fits"] and ok["pass_len"] == lp.PASS_MIN
    assert bad["passes"] and not bad["fits"] and bad["pass_len"] == lp.PASS_MIN


CASES = [  # H, B, capacity, seqlens
    (32, 9, 131072, [0, 1, 6399, 6400, 6401, 20000, 65535, 100000, 131071]),
    (64, 1, 262144, [262143]), (64, 1, 262144, [300]), (64, 1, 262144, [40000]),
    (28, 10, 43008, [43007, 0, 1, 17407, 17408, 30000, 511, 512, 25000, 40000]),
    (8, 1, 1 << 20, [(1 << 20) - 1]), (32, 4, 131072, [131071, 3, 33000, 60000]),
]


@pytest.mark.parametrize("wbits,hd", FMTS)
@pytest.mark.parametrize("H,B,ctx,seqlens", CASES)
def test_every_position_in_exactly_one_pass(wbits, hd, H, B, ctx, seqlens):
    """Each position of [0, seqlen] (the appended row included) falls in exactly one (chunk, pass); the staged window is in
    the first pass of its chunk, every pass's ring covers the rest of its cached rows, and the appended row is in the last
    pass of the last chunk."""
    p = lp.long_plan(wbits, hd, H, B, 1, ctx, seqlens)
    assert p["passes"] and p["nsplit"] == ar.nsplit_of(1, ctx, H, B)
    assert B * H * p["nsplit"] <= 2 * ar.H100_SMS or p["nsplit"] == 1
    for b, sl in enumerate(seqlens):
        cs = [c for c in p["ctas"] if c["b"] == b]
        cover = np.zeros(sl + 1, dtype=int)
        news = []
        for c in cs:
            for k, ps in enumerate(c["passes"]):
                assert 0 < ps["hi"] - ps["lo"] <= p["pass_len"]
                cover[ps["lo"]:ps["hi"]] += 1
                assert ps["n_st"] == (c["n_st"] if k == 0 else 0)
                beyond = ps["c_hi"] - ps["ring_lo"]
                assert ps["ntail"] * p["sub"] >= beyond > (ps["ntail"] - 1) * p["sub"] or (ps["ntail"] == 0 and beyond <= 0)
                if ps["new_row"]:
                    news.append((c["z"], k))
        assert (cover == 1).all()
        assert news == [(cs[-1]["z"], len(cs[-1]["passes"]) - 1)]


def test_boundary_needles_land_on_pass_edges():
    p = lp.long_plan(4, 128, 64, 1, 1, 131072, [131071])
    assert p["nsplit"] == 4 and [len(c["passes"]) for c in p["ctas"]] == [6, 6, 6, 6]
    pos = set(lp.boundary_positions(p, 0))
    for c in p["ctas"]:
        for ps in c["passes"]:
            assert {ps["lo"], ps["hi"] - 1} <= pos | {131071}
            for t in range(ps["ntail"]):                    # every ring sub-chunk edge
                s0 = ps["ring_lo"] + t * p["sub"]
                assert {s0, min(s0 + p["sub"], ps["c_hi"]) - 1} <= pos | {131071}
    assert {e + d for e in range(ar.PAGE, 131071, ar.PAGE) for d in (-1, 0)} <= pos      # every page edge
