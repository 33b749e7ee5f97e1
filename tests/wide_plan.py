"""Plain-Python restatement of the wide wgmma launch (csrc/gemm_tc.cu gemm_tc_launch and gemm_tc_kernel<32 / 64>, csrc/gemv.cuh,
csrc/qmatrix.cu qmatrix_chain_buffers): the token tile per row count, the shared-memory map and stage count, the split-K
workspace a launch needs, and the per-matrix and per-stream buffer sizes.  tests/test_wide_plan.py checks it, and pins every
constant below against its constexpr in the source."""
import math

GEMV_MTOK = 8
GEMV_MAX_CHAIN_ROWS = 64
TC_WARPS = 8
TC_MAX_STAGES = 4
TC_A_BUFS = 2
TC_A_BYTES = 128 * 32 * 2
TC_SMEM_BARS = (TC_WARPS * TC_MAX_STAGES + 2 * TC_MAX_STAGES) * 8
TC_SMEM_CAP = 200 * 1024
TC_WS_BYTES = 32 << 20
TC_WIDE_WS_BYTES = 96 << 20
TC_WIDE_XP_BYTES = 3 * 65536 * 128
SPLIT_F = 16                                  # per-segment fixed cost of the grid rule, in slabs
H100_SMS = 132


def tile_for(rows: int, chained: bool = True) -> int:
    """token tile of one launch: chained launches run all rows in one pass; others in 8-row passes.  Raises above 64."""
    if not chained or rows <= GEMV_MTOK:
        return GEMV_MTOK
    if rows > GEMV_MAX_CHAIN_ROWS:
        raise ValueError(f"a chained launch takes at most {GEMV_MAX_CHAIN_ROWS} rows")
    return 32 if rows <= 32 else 64


def act_stage(tw): return 128 * tw * 2
def misc_bytes(tw): return 128 + 4 * tw if tw > GEMV_MTOK else 128
def ssq_bytes(tw): return 4 * tw * 4
def corr_floats(tw): return 2 * 2 * 4 * 2 * tw
def red_floats(tw): return tw * 128
def comb_bytes(tw): return 2 * tw * 128 * 4 + tw * 128 * 2
def comb_overlaid(tw): return tw > GEMV_MTOK


def header_bytes(tw):
    raw = TC_SMEM_BARS + misc_bytes(tw) + (0 if comb_overlaid(tw) else comb_bytes(tw)) + ssq_bytes(tw) + corr_floats(tw) * 4
    return (raw + 1023) // 1024 * 1024


def ctas_per_sm(tw, tc_ctas=2):
    return 1 if tw > GEMV_MTOK else tc_ctas


def smem_plan(tw, stage_bytes, tc_ctas=2):
    """(stages, total bytes) of a launch whose largest group of a 32-column block is stage_bytes"""
    budget = min(227 * 1024 // ctas_per_sm(tw, tc_ctas) - 1024, TC_SMEM_CAP)
    def total(st):
        return header_bytes(tw) + 2 * TC_A_BUFS * TC_A_BYTES + st * (2 * act_stage(tw) + TC_WARPS * stage_bytes)
    st = TC_MAX_STAGES
    while st > 2 and total(st) > budget:
        st -= 1
    return st, total(st)


def block_bytes(bits): return 128 * bits          # 32 k x 32 columns


def stage_bytes_of(plan):
    """largest (slabs per group) x block bytes over a plan's regions; None when the kernel cannot stage it"""
    if plan[0] == "gptq":
        gs = plan[1]
        if gs <= 0 or gs > 128:
            return None
        return (gs // 32) * block_bytes(4)
    bits, _, gs = plan
    gss = gs if isinstance(gs, tuple) else (gs,) * len(bits)
    out = 0
    for b, g in zip(bits, gss):
        if g > 128 or (g // 32) * block_bytes(b) > 4096:
            return None
        out = max(out, (g // 32) * block_bytes(b))
    return out


def grid_rule(strips, KS, tw, sms=H100_SMS, tc_ctas=2):
    """(grid, maxc, aligned) of gemm_tc_launch for matrices of `strips` 128-column strips in total over K = 32 KS; aligned:
    every strip cut into S K-ranges (one segment per CTA) rather than plain stream-K over all resident slots"""
    units = strips * KS
    slots = sms * ctas_per_sm(tw, tc_ctas)
    grid = min(slots, units)
    L = -(-units // grid)
    cost_stream = (-(-L // KS) + 1) * SPLIT_F + L
    aligned = False
    if strips <= slots:
        S = min(slots // strips, max(1, KS // 8))
        if SPLIT_F + -(-KS // S) <= cost_stream:
            grid, aligned = strips * S, True
    grid = max(1, grid)
    return grid, KS * grid // units + 2, aligned


def grid_plan(strips, KS, tw, sms=H100_SMS, tc_ctas=2):
    """(grid, maxc) of gemm_tc_launch for matrices of `strips` 128-column strips in total over K = 32 KS"""
    return grid_rule(strips, KS, tw, sms, tc_ctas)[:2]


def ws_need(Ns, K, tw, sms=H100_SMS):
    """split-K workspace bytes of one launch over matrices of widths Ns sharing K"""
    strips = sum(-(-n // 128) for n in Ns)
    _, maxc = grid_plan(strips, K // 32, tw, sms)
    return strips * maxc * red_floats(tw) * 4


def launches(hidden, inter, heads, kv_heads, hd, vocab):
    """(name, widths, K) of every launch of a chained decode step"""
    return [("qkv", [heads * hd, kv_heads * hd, kv_heads * hd], hidden), ("o", [hidden], heads * hd),
            ("gate_up", [inter, inter], hidden), ("down", [hidden], inter), ("head", [vocab], hidden)]


PRESETS = {
    "7B": (4096, 11008, 32, 32, 128, 32000),
    "70B": (8192, 28672, 64, 8, 128, 32000),
    "TinyLlama": (2048, 5632, 32, 4, 64, 32000),
    "head152064": (3584, 18944, 28, 4, 128, 152064),
}


def chain_buffer_bytes(K, rows):
    """(activation buffer, sums of squares) bytes of a consumer matrix of K rows for a chained launch of `rows` rows"""
    slots = 64 if rows > GEMV_MTOK else 8
    return K * 2 * slots, (K // 128 + 2) * slots * 4


# ---- the per-CTA walk of gemm_tc_kernel: segments, group snapping, warpgroup halves and the split-K hand-off ----------------

def group_start(regions, KS, ks):
    """tc_group_start: the first slab of the group that holds slab ks (KS for ks >= KS); regions (ks_begin, bits, spg_log2)"""
    if ks >= KS:
        return KS
    kb, _, lg = [r for r in regions if r[0] <= ks][-1]
    return kb + (((ks - kb) >> lg) << lg)


def cta_of_unit(x, G, U):
    """tc_cta_of_unit: the CTA whose unit range [b U / G, (b + 1) U / G) holds unit x"""
    return ((x + 1) * G - 1) // U


def walk(mats, KS, G, paired=False):
    """Every segment the CTAs of a launch of G CTAs run, in the kernel's order.  mats: [(strips, regions)] sharing K = 32 KS.
    A segment: cta, mat (mi), strip, ks (the raw slab range), wg (the two warpgroups' snapped ranges), nc / jc (contributors
    of the strip and this CTA's workspace slot), slot (its strip's global index, gs), counter (cidx) and expected."""
    U = sum(s for s, _ in mats) * KS
    ub, sb0 = [], []
    for s, _ in mats:
        ub.append(sum(m[0] for m in mats[:len(ub)]) * KS)
        sb0.append(sum(m[0] for m in mats[:len(sb0)]))
    ncs = lambda m, strip: cta_of_unit(ub[m] + strip * KS + KS - 1, G, U) - cta_of_unit(ub[m] + strip * KS, G, U) + 1
    out = []
    for b in range(G):
        u, u1 = b * U // G, (b + 1) * U // G
        while u < u1:
            mi = 0
            while mi + 1 < len(mats) and u >= ub[mi + 1]:
                mi += 1
            regions = mats[mi][1]
            local = u - ub[mi]
            strip, ks_a = divmod(local, KS)
            seg = min(KS - ks_a, u1 - u)
            ks0, ks1 = group_start(regions, KS, ks_a), group_start(regions, KS, ks_a + seg)
            ksm = group_start(regions, KS, ks0 + ((ks1 - ks0 + 1) >> 1))
            nc = ncs(mi, strip)
            jc = b - cta_of_unit(ub[mi] + strip * KS, G, U)
            expected, counter = nc, sb0[mi] + strip
            if paired:
                expected += ncs(1 - mi, strip)
                counter = sb0[0] + strip
            out.append(dict(cta=b, mat=mi, strip=strip, ks=(ks_a, ks_a + seg), wg=((ks0, ksm), (ksm, ks1)), nc=nc, jc=jc,
                            slot=sb0[mi] + strip, counter=counter, expected=expected, alone=nc == 1 and not paired))
            u += seg
    return out


def regimes(segs, G):
    """what a launch's walk reaches: most segments in one CTA, CTAs whose segments cross from one matrix to the next, segments
    whose snapped range is empty, and segments where one warpgroup gets no group"""
    per = [[s for s in segs if s["cta"] == b] for b in range(G)]
    return dict(
        max_segs=max(len(p) for p in per),
        crossings=sum(len({s["mat"] for s in p}) > 1 for p in per),
        empty_segs=sum(s["wg"][0][0] == s["wg"][1][1] for s in segs),
        empty_wg=sum(s["wg"][0][0] < s["wg"][1][1] and (s["wg"][0][0] == s["wg"][0][1] or s["wg"][1][0] == s["wg"][1][1])
                     for s in segs))


# ---- the launches of tests/test_gpu_wide_full_shapes.py ------------------------------------------------------------------------

M54 = ((5, 4), (0.1, 0.9), 128)                   # model.py _mix_4bpw
M43 = ((4, 3), (0.1, 0.9), 128)
HEAD6 = ((6,), (1.0,), 128)
HEAD8 = ((8,), (1.0,), 128)                       # the 8-bit head of the exl2-8bpw test model: 4 KB stages
GPTQ = ("gptq", 128, True)
A70, M70 = ((4, 3), (0.1, 0.9), 128), ((3, 2), (0.3, 0.7), 64)    # model.py llama2-70b-2.5bpw

# block: (hidden, inter, heads, kv_heads, attention plan, MLP plans, heads: [(vocab, plan)])
FULL_BLOCKS = {
    "7b-4.0bpw": (4096, 11008, 32, 32, M54, [M54, M43], [(32000, HEAD6), (32000, HEAD8)]),
    "7b-gptq": (4096, 11008, 32, 32, GPTQ, [GPTQ], [(32000, HEAD6)]),
    "70b-2.5bpw": (8192, 28672, 64, 8, A70, [M70], [(32000, HEAD6), (152064, HEAD6)]),
}


def block_launches(block):
    """(name, [(N, plan)], K, paired) of every chained launch a block's step makes"""
    hid, inter, H, KVH, ap, mps, heads = FULL_BLOCKS[block]
    out = [("qkv", [(H * 128, ap), (KVH * 128, ap), (KVH * 128, ap)], hid, False), ("o", [(hid, ap)], H * 128, False)]
    for i, mp in enumerate(mps):
        out += [(f"gate_up{i}", [(inter, mp), (inter, mp)], hid, True), (f"down{i}", [(hid, mp)], inter, False)]
    out += [(f"head{n}_{p[0][0]}", [(n, p)], hid, False) for n, p in heads]
    return out


def launch_walk(Ns, K, paired, tw=32, regions_of=None):
    """(grid, maxc, aligned, segments) of one launch; regions_of(K, plan) gives a matrix's regions (tests/i8_plans.py)"""
    if regions_of is None:
        from i8_plans import regions_of
    strips = [-(-n // 128) for n, _ in Ns]
    KS = K // 32
    G, maxc, aligned = grid_rule(sum(strips), KS, tw)
    return G, maxc, aligned, walk([(s, regions_of(K, p)) for s, (_, p) in zip(strips, Ns)], KS, G, paired)
