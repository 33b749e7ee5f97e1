"""CPU emulation of the index / byte-order logic of csrc/gemv_i8.cu (no GPU): the parts of the batch-1 integer GEMV
that are pure bookkeeping and that a wrong constant would break silently.

1. consume_slab: for every bit width, compose a 32 k x 32 column block in the TC layout (layout.h
   compose_lane_words), stage a row of 16-bit integers in the order stage_round writes it (high / low byte planes,
   bytes of octet j ordered k = 8j + {0,4,1,5} | {2,6,3,7}) and run the kernel's mask / shift sequence (no operand is permuted:
   layout.h pair_word / pair_slot give every plane the same byte order); the
   integer sums must equal sum_k a_k q_k exactly.
2. work split: the host-side block -> CTA partition (whole 32-column blocks per CTA, balanced by bytes).
"""
import numpy as np
import pytest

# ---- layout.h ---------------------------------------------------------------------------------------------------------


def plane_main(b):
    return {2: 2, 3: 2, 8: 8}.get(b, 4)


def plane_extra(b):
    return {3: 1, 5: 1, 6: 2}.get(b, 0)


def pair_word(P, p):
    return {4: p // 4, 2: p >> 3, 1: 0, 8: 2 * (p >> 2) + (p & 1)}[P]


def pair_slot(P, p):
    return {4: p % 4, 2: 4 * ((p >> 1) & 1) + 2 * ((p & 7) >> 2) + (p & 1), 1: 8 * ((p >> 1) & 1) + 2 * (p >> 2) + (p & 1),
            8: (p >> 1) & 1}[P]


def compose_lane_words(bits, q):
    """q: 32 values of one column (k = 0..31) -> (main words, extra words) exactly as layout.h compose_lane_words."""
    Pm, Pe = plane_main(bits), plane_extra(bits)
    mw = [0] * Pm
    ew = [0] * Pe
    for i in range(32):
        p, e = i >> 1, i & 1
        fm = int(q[i]) & ((1 << Pm) - 1)
        mw[pair_word(Pm, p)] |= fm << (16 * e + Pm * pair_slot(Pm, p))
        if Pe:
            fe = (int(q[i]) >> Pm) & ((1 << Pe) - 1)
            ew[pair_word(Pe, p)] |= fe << (16 * e + Pe * pair_slot(Pe, p))
    return [w & 0xFFFFFFFF for w in mw], [w & 0xFFFFFFFF for w in ew]


# ---- gemv_i8.cu --------------------------------------------------------------------------------------------------------


def dp4a(w, x, signed_x):
    s = 0
    for i in range(4):
        wb = (w >> (8 * i)) & 0xFF
        xb = (x >> (8 * i)) & 0xFF
        if signed_x and xb >= 128:
            xb -= 256
        s += wb * xb
    return s


def stage_row(a):
    """a: 32 int16 values (one slab) -> XH[8], XL[8] as stage_round packs them."""
    XH, XL = [0] * 8, [0] * 8
    for j in range(4):
        q = [int(v) for v in a[8 * j:8 * j + 8]]

        def pack(idx, sh):
            w = 0
            for n, i in enumerate(idx):
                w |= ((q[i] >> sh) & 0xFF) << (8 * n)
            return w
        XH[2 * j], XH[2 * j + 1] = pack((0, 4, 1, 5), 8), pack((2, 6, 3, 7), 8)
        XL[2 * j], XL[2 * j + 1] = pack((0, 4, 1, 5), 0), pack((2, 6, 3, 7), 0)
    return XH, XL


def consume_slab(bits, mw, ew, XH, XL):
    """One column of consume_slab<BITS>; returns the value the flush computes before the zero-point term."""
    Pm, Pe = plane_main(bits), plane_extra(bits)
    am = [0, 0, 0, 0]
    ae = [0, 0]
    if Pm == 4:
        for j in range(4):
            lo, hi = mw[j] & 0x0F0F0F0F, mw[j] & 0xF0F0F0F0
            am[0] += dp4a(lo, XH[2 * j], True)
            am[1] += dp4a(lo, XL[2 * j], False)
            am[2] += dp4a(hi, XH[2 * j + 1], True)
            am[3] += dp4a(hi, XL[2 * j + 1], False)
    elif Pm == 8:
        for w in range(8):
            am[0] += dp4a(mw[w], XH[w], True)
            am[1] += dp4a(mw[w], XL[w], False)
    else:
        for w in range(2):
            for i in range(4):
                t = (mw[w] >> (2 * i)) & 0x03030303
                am[0] += dp4a(t, XH[w * 4 + i], True)
                am[1] += dp4a(t, XL[w * 4 + i], False)
    if Pe == 1:
        for i in range(8):
            f = (ew[0] >> i) & 0x01010101
            ae[0] += dp4a(f, XH[i], True)
            ae[1] += dp4a(f, XL[i], False)
    elif Pe == 2:
        for w in range(2):
            for i in range(4):
                t = (ew[w] >> (2 * i)) & 0x03030303
                ae[0] += dp4a(t, XH[w * 4 + i], True)
                ae[1] += dp4a(t, XL[w * 4 + i], False)
    hi16 = (am[2] << 8) + am[3]
    assert hi16 % 16 == 0
    return ((am[0] << 8) + am[1]) + (hi16 >> 4) + (((ae[0] << 8) + ae[1]) << Pm)


@pytest.mark.parametrize("bits", [2, 3, 4, 5, 6, 8])
def test_consume_slab_selectors(bits):
    rng = np.random.default_rng(bits)
    for trial in range(20):
        q = rng.integers(0, 1 << bits, size=32)
        a = rng.integers(-32767, 32768, size=32)
        if trial == 0:
            a[:] = 0
            a[trial % 32] = 1
        mw, ew = compose_lane_words(bits, q)
        XH, XL = stage_row(a)
        got = consume_slab(bits, mw, ew, XH, XL)
        assert got == int((a.astype(np.int64) * q.astype(np.int64)).sum())


def test_consume_slab_one_hot_every_k():
    """every k position reaches its own weight (one-hot rows), all bit widths"""
    rng = np.random.default_rng(0)
    for bits in (2, 3, 4, 5, 6, 8):
        q = rng.integers(0, 1 << bits, size=32)
        mw, ew = compose_lane_words(bits, q)
        for k in range(32):
            a = np.zeros(32, dtype=np.int64)
            a[k] = -12345
            XH, XL = stage_row(a)
            assert consume_slab(bits, mw, ew, XH, XL) == -12345 * int(q[k])


# ---- work split ------------------------------------------------------------------------------------------------------------
# A CTA owns whole 32-column blocks; the block -> CTA table is computed on the host (gemv_i8.cu i8_partition_blocks) and is
# reachable without a GPU through the diagnostics hook exl2b_debug_partition.


def _partition(block_bytes, ctas):
    import ctypes

    from exllamav2_b200 import ext as ext_c
    f = ext_c.lib.exl2b_debug_partition
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    bb = np.asarray(block_bytes, dtype=np.uint32)
    out = np.zeros(ctas + 2, dtype=np.uint16)
    used = ctypes.c_int(0)
    rc = f(bb.ctypes.data, len(bb), ctas, out.ctypes.data, ctypes.byref(used))
    assert rc == 0
    return out[: used.value + 1].astype(int), used.value


def _best_makespan(block_bytes, ctas):
    """optimal contiguous partition by dynamic programming (small inputs only)"""
    n = len(block_bytes)
    pre = np.concatenate([[0], np.cumsum(block_bytes)])
    INF = float("inf")
    dp = [[INF] * (n + 1) for _ in range(ctas + 1)]
    dp[0][0] = 0
    for c in range(1, ctas + 1):
        for j in range(n + 1):
            dp[c][j] = dp[c - 1][j]
            for i in range(j):
                dp[c][j] = min(dp[c][j], max(dp[c - 1][i], pre[j] - pre[i]))
    return dp[ctas][n]


PART_CASES = [
    ("qkvo 128 blocks", [65536] * 128, 148),
    ("qkv fused [5,4] + [4] + [6,5,4]", [67584] * 128 + [65536] * 128 + [70000] * 128, 148),
    ("gate|up", [60000] * 344 + [60000] * 344, 148),
    ("head", [98304] * 1000, 148),
    ("one block", [4096], 148),
    ("three ragged", [4096, 4096, 2048], 148),
    ("more ctas than blocks", [1000] * 7, 148),
    ("few ctas", [10, 20, 30, 40, 50, 60, 70, 80, 90, 100, 5, 5], 4),
]


@pytest.mark.parametrize("name,bb,ctas", PART_CASES, ids=[c[0] for c in PART_CASES])
def test_block_partition(name, bb, ctas):
    bounds, used = _partition(bb, ctas)
    assert 1 <= used <= ctas
    assert bounds[0] == 0 and bounds[-1] == len(bb)
    assert all(b > a for a, b in zip(bounds, bounds[1:])), "every CTA in use owns at least one block, in order"
    pre = np.concatenate([[0], np.cumsum(bb)])
    worst = max(pre[b] - pre[a] for a, b in zip(bounds, bounds[1:]))
    total, biggest = int(pre[-1]), max(bb)
    assert worst >= max(biggest, -(-total // ctas))
    if len(bb) <= 16:
        assert worst == _best_makespan(bb, ctas)
    else:
        # uniform-ish blocks: never more than one block above the ideal share
        assert worst <= -(-total // ctas) + biggest


# ---- stage lists -----------------------------------------------------------------------------------------------------------
# gemv_i8.cu i8_build_lists (host): every (block, slab) unit of the launch appears in exactly one stage of exactly one warp, in
# order; a stage never crosses a quantisation group, a 128-k row block, a bit-width region, and fits the ring slot; the flush
# flag closes every group / row block / range, the block-done flag the warp's share of a block.


def _plan(N, KS, regions, ctas=148, warps=16, slot=6144, gptq=0):
    import ctypes

    from exllamav2_b200 import ext as ext_c
    f = ext_c.lib.exl2b_debug_plan
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                  ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    # regions: (ks_begin, bits, spg_log2); group_base / off_base derived like qmatrix.cu build_regions
    reg, gbase, off = [], 0, 0
    for i, (ks0, bits, lg) in enumerate(regions):
        ks1 = regions[i + 1][0] if i + 1 < len(regions) else KS
        reg += [ks0, bits, lg, gbase, off]
        gbase += -(-(ks1 - ks0) // (1 << lg))
        off += (ks1 - ks0) * 128 * bits
    stream_bytes = off
    ra = np.asarray(reg, dtype=np.int32)
    cap = ((N + 31) // 32) * KS + 148 * 16 * 8
    desc = np.zeros((cap, 4), dtype=np.uint32)
    first = np.zeros(ctas * warps + 2, dtype=np.uint32)
    used, nd, lcap = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_int(0)
    red = np.zeros((N + 31) // 32, dtype=np.uint32)
    rc = f(N, KS, gptq, stream_bytes, ra.ctypes.data, len(regions), ctas, warps, slot, desc.ctypes.data, cap, first.ctypes.data,
           ctypes.byref(used), ctypes.byref(nd), ctypes.byref(lcap), red.ctypes.data)
    assert rc == 0
    return desc[: nd.value], first[: used.value * warps + 1], used.value, lcap.value, stream_bytes, reg, red


PLAN_CASES = [
    ("4096x4096 [5,4] g128", 4096, 128, [(0, 5, 2), (13, 4, 2)]),
    ("11008 cols [4,3] g128", 11008, 128, [(0, 4, 2), (13, 3, 2)]),
    ("K=11008 [5,4]", 4096, 344, [(0, 5, 2), (36, 4, 2)]),
    ("head 6-bit", 32000, 128, [(0, 6, 2)]),
    ("8-bit g32 + 2-bit g64", 512, 64, [(0, 8, 0), (5, 2, 1)]),
    ("g256", 1024, 64, [(0, 4, 3)]),
    ("ragged columns", 1000, 16, [(0, 3, 0), (3, 2, 2)]),
    ("fewer slabs than warps", 64, 8, [(0, 4, 2)]),
]


@pytest.mark.parametrize("name,N,KS,regions", PLAN_CASES, ids=[c[0] for c in PLAN_CASES])
@pytest.mark.parametrize("warps,slot", [(16, 6144), (12, 4096), (16, 2048)])
def test_stage_lists(name, N, KS, regions, warps, slot):
    desc, first, C, lcap, stream_bytes, reg, red = _plan(N, KS, regions, warps=warps, slot=slot)
    partials = {}          # block -> [(warp, partial slot)] as the kernel's main loop leaves them
    nblk = (N + 31) // 32
    seen = np.zeros((nblk, KS), dtype=np.int32)
    n_pre_all = (first >> 26).astype(int)
    first = first & 0x3FFFFFF
    assert first[0] == 0 and first[-1] == len(desc) and np.all(np.diff(first.astype(np.int64)) >= 0)
    assert lcap == int(np.max(np.diff(first.astype(np.int64))))
    # CTA block ranges: recover from the partition hook (same inputs)
    bounds, used = _partition([stream_bytes] * nblk, 148)
    assert used == C
    ends = {r[0]: (regions[i + 1][0] if i + 1 < len(regions) else KS) for i, r in enumerate(regions)}
    for c in range(C):
        for w in range(warps):
            lst = desc[first[c * warps + w]: first[c * warps + w + 1]]
            # the arena (`slot` bytes per warp) as the kernel drives it: stages are requested up front / as space frees, never over
            # a stage that has not been consumed, at most 8 in flight (one mbarrier each), and always before they are waited for
            requested, live = n_pre_all[c * warps + w], {}
            sizes = [int(((z >> 11) & 7) * ((z >> 14) & 15) * 128) for (_, _, z, _) in lst]
            offs = [int((bw >> 16) & 0xFF) * 128 for (_, _, _, bw) in lst]

            def request(sidx):
                assert offs[sidx] + sizes[sidx] <= slot
                for j, (o, sz) in live.items():
                    assert offs[sidx] + sizes[sidx] <= o or o + sz <= offs[sidx], "arena overlap with an unconsumed stage"
                    assert j % 8 != sidx % 8, "mbarrier still in use"
                live[sidx] = (offs[sidx], sizes[sidx])
            for sidx in range(min(requested, len(lst))):
                request(sidx)
            assert requested <= len(lst) and (requested >= 1 or len(lst) == 0)
            for cidx in range(len(lst)):
                assert cidx < requested, "stage waited for before it was requested"
                del live[cidx]
                for _ in range(int((lst[cidx][3] >> 24) & 15)):
                    request(requested)
                    requested += 1
            assert requested == len(lst)
            prev = None
            blk_slabs = emits = 0
            for i, (x, y, z, bw) in enumerate(lst):
                ks, n, bits, flags, mi = z & 0x7FF, (z >> 11) & 7, (z >> 14) & 15, (z >> 18) & 15, (z >> 22) & 3
                blk = bounds[c] + int(bw & 0xFFFF)
                assert mi == 0 and 1 <= n <= 4 and (n == 1 or n * bits * 128 <= slot // 2)
                r = max(j for j, rg in enumerate(regions) if ks >= rg[0])
                ks0, rb, lg = regions[r]
                assert bits == rb and ks + n <= ends[ks0], "one region"
                assert (ks >> 2) == ((ks + n - 1) >> 2), "one 128-k row block"
                g0, g1 = (ks - ks0) >> lg, (ks + n - 1 - ks0) >> lg
                assert g0 == g1, "one group"
                assert x == blk * stream_bytes + reg[5 * r + 4] + (ks - ks0) * 128 * bits
                assert y == (reg[5 * r + 3] + g0) * N + blk * 32
                seen[blk, ks:ks + n] += 1
                cur = (blk, ks)
                if prev is not None:
                    assert cur == (prev[0], prev[1]) or cur == (prev[0] + 1, 0), "contiguous walk"
                prev = (blk, ks + n) if ks + n < KS else (blk + 1, 0)
                last = i + 1 == len(lst)
                nxt = lst[i + 1] if not last else None
                group_closes = last or ks + n == KS or ((ks + n) & 3) == 0 or ks + n == ends[ks0] or ((ks + n - ks0) >> lg) != g0
                assert bool(flags & 1) == group_closes, "flush flag"
                assert bool(flags & 2) == (last or ks + n == KS), "block-done flag"
                assert not (flags & 4)
                blk_slabs += n
                if flags & 2:
                    if blk_slabs != KS:
                        assert emits < 2
                        partials.setdefault(blk, []).append((w, emits))
                        emits += 1
                    blk_slabs = 0
    assert np.all(seen == 1), "every (block, slab) exactly once"
    # the table the launch's tail reads: the warps that hold a partial sum of each block, and the first one's slot
    for blk in range(nblk):
        ps = partials.get(blk, [])
        mask = 0
        for (w, _) in ps:
            mask |= 1 << w
        assert int(red[blk]) & 0xFFFF == mask
        if ps:
            assert (int(red[blk]) >> 16) & 1 == ps[0][1] and all(sl == 0 for (_, sl) in ps[1:])
            assert [w for (w, _) in ps] == sorted(w for (w, _) in ps)


# ---- row quantisation ------------------------------------------------------------------------------------------------------
# gemv_i8.cu stage_round, restated in numpy: per 128-k block the row becomes 16-bit integers with a power-of-two scale whose
# exponent is taken from max * (1 + 2^-15); rounding is done by the fp32 adder (x * inv + 1.5 * 2^23, low 16 bits = int16).


def quantise_block(f):
    """f: 128 float32 values -> (int array q, float32 scale) exactly as the kernel computes them."""
    f = f.astype(np.float32)
    amax = np.float32(np.max(np.abs(f)))
    if amax == 0:
        return np.zeros(128, dtype=np.int64), np.float32(0)
    ef = (np.float32(amax * np.float32(1.000030518)).view(np.uint32) >> 23) & 0xFF
    inv = np.uint32((268 - int(ef)) << 23).view(np.float32)
    bits = (f * inv + np.float32(12582912.0)).astype(np.float32).view(np.uint32)           # fma in the kernel: x * inv is exact (power of two)
    q = (bits & 0xFFFF).astype(np.int64)
    q = np.where(q >= 32768, q - 65536, q)
    scale = np.uint32((int(ef) - 14) << 23).view(np.float32)
    return q, scale


def test_row_quantisation_range_and_rounding():
    rng = np.random.default_rng(0)
    for trial in range(300):
        f = rng.standard_normal(128).astype(np.float32) * np.float32(10.0 ** rng.uniform(-6, 4))
        if trial % 3 == 0:      # adversarial maxima: mantissas at the top of a binade (would round up to 2^15 without the bump)
            f[rng.integers(128)] = np.float32(np.nextafter(np.float32(2.0 ** rng.integers(-20, 15)), np.float32(0)))
        q, scale = quantise_block(f)
        assert q.min() >= -32767 and q.max() <= 32767, "int16 high byte must keep its sign"
        amax = np.max(np.abs(f))
        assert np.max(np.abs(q)) >= 8192, "the block maximum uses at least 14 bits"
        # round-to-nearest-even of x / scale, error <= half a step = 2^-15 .. 2^-14 of the block maximum
        ref = np.rint(f.astype(np.float64) / float(scale)).astype(np.int64)
        assert np.array_equal(q, ref)
        assert np.max(np.abs(q * float(scale) - f.astype(np.float64))) <= 0.5 * float(scale) * (1 + 1e-12)
        assert 0.5 * float(scale) <= amax * 2.0 ** -14


def test_row_quantisation_exact_for_fp16_within_16x_of_the_maximum():
    """fp16 inputs within a factor 16 of their block's maximum are represented exactly (an 11-bit significand fits above the 2^-14
    step): a unit-vector row therefore returns reconstruct()'s fp16 weights bit for bit."""
    rng = np.random.default_rng(1)
    for _ in range(100):
        e = rng.integers(-8, 8)
        f = (rng.uniform(1.0 / 16, 1.0, 128) * rng.choice([-1, 1], 128) * 2.0 ** e).astype(np.float16).astype(np.float32)
        f[0] = np.float32(np.float16(2.0 ** e * 0.999))
        q, scale = quantise_block(f)
        assert np.array_equal((q * float(scale)).astype(np.float32), f)
