"""The long-context regime of the fused K/V-cache decode attention (csrc/attn_q4.cu attn_launch_plan, pass_len, and
attn_q4_passes_kernel), restated in Python on top of tests/attn_regimes.py.

A single-token decode launch whose whole-chunk score buffer does not fit the 200 KB shared-memory limit walks each CTA's
positions in passes of at most `pass_len` positions, with an online softmax across them.  Every other launch keeps the plan
attn_regimes.plan() restates.  `long_plan()` says which regime a launch takes, its pass length and footprint, and each
working CTA's passes: the positions of each, the staged window (first pass only) and the ring sub-chunks that stream the
rest.  tests/test_attn_long_plan.py pins it; tests/test_gpu_attn_long_context.py takes its capacities and needle positions
from it.
"""
from __future__ import annotations

import attn_regimes as ar

# attn_q4.cu: AQ_PASS_SMEM, AQ_PASS_MIN, AQ_PASS_ALIGN
PASS_SMEM = 114 * 1024        # target footprint: 228 KB per SM - 111 KB GEMV CTA - 2 x 1 KB reserved - 1 KB static + slack
PASS_MIN = 512                # the shortest pass; a page table that leaves no room for it is refused
PASS_ALIGN = 256              # pass lengths are multiples of 256 positions (whole pages at the default page size)


def _score_bytes(sc_len: int) -> int:
    return ((sc_len + 3) & ~3) * 4


def long_plan(wbits: int, hd: int, H: int, B: int, q_len: int, max_ctx: int, seqlens=None, sms: int = ar.H100_SMS,
              page_size: int = ar.PAGE) -> dict:
    """The launch `exl2b_paged_attn_decode_q` makes: attn_regimes' plan, and whether it walks its positions in passes.

    Returns nsplit, passes (the regime is taken), pass_len (0 without passes), smem (the launch's dynamic shared memory),
    fits (smem <= 200 KB: the launch is accepted), stage, sub, and with `seqlens` the list `ctas`: attn_regimes.plan()'s
    CTAs, each with `passes`, a list of dicts
      lo, hi       the positions of the pass, [lo, hi); scores sit in sc[p - lo]
      c_hi         the end of its cached rows, min(hi, seqlen)
      n_st         staged rows, [lo, lo + n_st) (the CTA's staged window, first pass only)
      ring_lo      the first row streamed through the ring, lo + n_st
      ntail        ring sub-chunks of `sub` positions from ring_lo on
      new_row      the appended row (position seqlen) is scored in this pass"""
    nsplit = ar.nsplit_of(q_len, max_ctx, H, B, sms)
    base = ar.smem_bytes(wbits, hd, q_len, max_ctx, nsplit, page_size)
    out = dict(nsplit=nsplit, passes=False, pass_len=0, smem=base["smem"], fits=base["fits"], stage=base["stage"],
               sub=base["sub"], ring=base["ring"])
    if q_len == 1 and not base["fits"]:
        assert base["ring"]
        rest = base["smem"] - _score_bytes(base["sc_len"])            # attn_smem_map with sc_len = 0
        room = max(0, PASS_SMEM - rest) // 4
        pass_len = max(PASS_MIN, room // PASS_ALIGN * PASS_ALIGN)
        smem = rest + _score_bytes(pass_len)
        out.update(passes=True, pass_len=pass_len, smem=smem, fits=smem <= ar.SMEM_LIMIT)
    if seqlens is None:
        return out
    p = ar.plan(wbits, hd, H, B, q_len, max_ctx, seqlens, sms, page_size)
    assert p["nsplit"] == nsplit and p["stage"] == out["stage"] and p["sub"] == out["sub"]
    out["ctas"] = []
    for c in p["ctas"]:
        c = dict(c)
        step = out["pass_len"] if out["passes"] else c["p_hi"] - c["p_lo"]
        c["passes"] = []
        for lo in range(c["p_lo"], c["p_hi"], max(1, step)):
            hi = min(c["p_hi"], lo + step)
            c_hi = min(hi, c["seqlen"])
            n_st = c["n_st"] if lo == c["p_lo"] else 0
            beyond = max(0, c_hi - lo - n_st)
            ntail = -(-beyond // out["sub"]) if out["ring"] else 0
            c["passes"].append(dict(lo=lo, hi=hi, c_hi=c_hi, n_st=n_st, ring_lo=lo + n_st, ntail=ntail,
                                    new_row=lo <= c["seqlen"] < hi))
        out["ctas"].append(c)
    return out


def largest_fit(wbits: int, hd: int, H: int, B: int, q_len: int = 1, page_size: int = ar.PAGE) -> int:
    """The largest capacity (positions, whole pages) whose launch takes today's single-pass plan."""
    pages = 1
    while ar.smem_bytes(wbits, hd, q_len, (pages + 1) * page_size,
                        ar.nsplit_of(q_len, (pages + 1) * page_size, H, B))["fits"]:
        pages += 1
    return pages * page_size


def largest_page_table(wbits: int, hd: int, H: int = 8, B: int = 1, page_size: int = ar.PAGE) -> int:
    """The most pages per sequence a single-token launch accepts: the page table plus a pass of PASS_MIN positions fit 200 KB."""
    lo, hi = 1, 1 << 16
    while lo + 1 < hi:                # long_plan(...)["fits"] holds at lo and fails at hi
        mid = (lo + hi) // 2
        if long_plan(wbits, hd, H, B, 1, mid * page_size, page_size=page_size)["fits"]:
            lo = mid
        else:
            hi = mid
    return lo


def boundary_positions(lp: dict, b: int, page_size: int = ar.PAGE) -> list:
    """Cached positions of sequence b where the passes regime goes wrong first: both sides of every pass and chunk edge,
    the end of the staged window, both sides of every ring sub-chunk edge of every pass, and both sides of every page edge."""
    pos = set()
    seqlen = None
    for c in lp["ctas"]:
        if c["b"] != b:
            continue
        seqlen = c["seqlen"]
        pos.update({c["p_lo"], c["p_hi"] - 1})
        for ps in c["passes"]:
            pos.update({ps["lo"], ps["lo"] + 1, ps["hi"] - 2, ps["hi"] - 1, ps["ring_lo"] - 1, ps["ring_lo"]})
            for t in range(ps["ntail"]):
                s0 = ps["ring_lo"] + t * lp["sub"]
                pos.update({s0, s0 + lp["sub"] - 1})
    if seqlen is None:
        return []
    for e in range(page_size, seqlen + 1, page_size):
        pos.update({e - 1, e})
    pos.add(seqlen - 1)
    return sorted(x for x in pos if 0 <= x < seqlen)
