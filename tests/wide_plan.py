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


def grid_plan(strips, KS, tw, sms=H100_SMS, tc_ctas=2):
    """(grid, maxc) of gemm_tc_launch for matrices of `strips` 128-column strips in total over K = 32 KS"""
    units = strips * KS
    slots = sms * ctas_per_sm(tw, tc_ctas)
    grid = min(slots, units)
    L = -(-units // grid)
    cost_stream = (-(-L // KS) + 1) * SPLIT_F + L
    if strips <= slots:
        S = min(slots // strips, max(1, KS // 8))
        if SPLIT_F + -(-KS // S) <= cost_stream:
            grid = strips * S
    grid = max(1, grid)
    return grid, KS * grid // units + 2


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
