"""The 8-bit K/V cache oracle (tests/kv_q68.py) against the reference extension's own Q6 / Q8 pack and unpack, stored in
tests/golden/ref_kv_q68.npz (tools/gen_golden_kv_q68.py):
  * pack: scales bit-exact; bytes equal except where the GPU's __h2div (reciprocal based) and the oracle's exact division
    round to different sides of a quantisation step -- those differ by exactly 1, in a small measured fraction;
  * unpack of the reference's bytes: bit-exact;
  * Q8's round-trip error on N(0, 1) rows is far below Q4's.
CPU only: no GPU needed."""
import os

import numpy as np
import pytest

import exl2_oracle as oracle
import kv_q68

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_kv_q68.npz")
# measured: on these cases no element differs (Q4 on N(0,1) rows: up to ~1e-3 of nibbles, test_kv_q4_roundtrip_nonpaged);
# the bound allows the same rare +-1 for other inputs
MAX_OFF_BY_ONE = 2e-3


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLDEN)


def _elements(q, bits):
    """uint8 state -> one integer per value."""
    q = np.asarray(q, dtype=np.uint8)
    if bits == 8:
        return q.astype(np.int32)
    out = np.empty(q.shape[:-1] + (q.shape[-1] * 2,), dtype=np.int32)
    out[..., 0::2], out[..., 1::2] = q & 15, q >> 4
    return out


def _check_pack(x, want_q, want_s, bits):
    q, s = kv_q68.kv_pack(x, bits)
    assert np.array_equal(np.asarray(s, dtype=np.float16).view(np.uint16), want_s), "scales differ"
    d = _elements(q, bits) - _elements(want_q, bits)
    assert np.abs(d).max() <= 1
    assert np.count_nonzero(d) <= MAX_OFF_BY_ONE * d.size, np.count_nonzero(d) / d.size


@pytest.mark.parametrize("wbits", [6, 8])
@pytest.mark.parametrize("name", list(kv_q68.NONPAGED))
def test_nonpaged_pack_unpack_vs_reference(gold, name, wbits):
    kb, vb = kv_q68.widths(wbits)
    k, v = kv_q68.nonpaged_inputs(name)
    a, b = kv_q68.nonpaged_range(name)
    tag = f"{name}_w{wbits}_"
    for x, item, bits in ((k, "k", kb), (v, "v", vb)):
        want_q, want_s = gold[tag + item + "q"], gold[tag + item + "s"]
        B, S = x.shape[:2]
        flat = lambda t: t.reshape(B, S, -1)
        # inside the range: the oracle's pack; outside: untouched (zero-initialised)
        _check_pack(flat(x)[:, a:b], flat(want_q)[:, a:b], flat(want_s)[:, a:b], bits)
        assert not flat(want_q)[:, :a].any() and not flat(want_q)[:, b:].any()
        assert not flat(want_s)[:, :a].any() and not flat(want_s)[:, b:].any()
        # unpack of the reference's bytes over the same range, bit-exact
        o = np.zeros_like(x).reshape(B, S, -1)
        o[:, a:b] = kv_q68.kv_unpack(flat(want_q)[:, a:b], flat(want_s)[:, a:b].view(np.float16), bits)
        assert np.array_equal(kv_q68.digest(o.reshape(x.shape)), gold[tag + item + "o"]), "unpack is not bit-exact"


@pytest.mark.parametrize("wbits", [6, 8])
@pytest.mark.parametrize("name", list(kv_q68.PAGED))
def test_paged_pack_unpack_vs_reference(gold, name, wbits):
    c = kv_q68.PAGED[name]
    kb, vb = kv_q68.widths(wbits)
    k, v = kv_q68.paged_inputs(name)
    rows = kv_q68.paged_rows(name)
    pg = np.array([r[2] for r in rows])
    rr = np.array([r[3] for r in rows])
    tag = f"{name}_w{wbits}_"
    for x, item, bits in ((k, "k", kb), (v, "v", vb)):
        want_q, want_s = gold[tag + item + "q_rows"], gold[tag + item + "s_rows"]
        _check_pack(x[pg, rr], want_q, want_s, bits)
        # the gathered rows are everything the pack wrote: rebuilt into zero tensors they give the stored whole-tensor digests
        q_all = np.zeros(x.shape[:-1] + (x.shape[-1] * bits // 8,), dtype=np.uint8)
        s_all = np.zeros(x.shape[:-1] + (x.shape[-1] // 32,), dtype=np.uint16)
        q_all[pg, rr], s_all[pg, rr] = want_q, want_s
        assert np.array_equal(kv_q68.digest(q_all), gold[tag + item + "q"])
        assert np.array_equal(kv_q68.digest(s_all), gold[tag + item + "s"])
        # unpack over [0, seqlen + q_len) of every sequence (widened to 512-value blocks), bit-exact
        o = np.zeros_like(x)
        dim = c["heads"] * c["hd"]
        for s, sl in enumerate(c["seqlens"]):
            n = ((sl + c["q_len"]) * dim + 511) // 512 * 512 if dim % 512 else (sl + c["q_len"]) * dim
            for tok in range((n + dim - 1) // dim):
                p, r = c["block_table"][s][tok // kv_q68.PAGE], tok % kv_q68.PAGE
                o[p, r] = kv_q68.kv_unpack(q_all[p, r].reshape(1, -1), s_all[p, r].view(np.float16).reshape(1, -1), bits).reshape(o[p, r].shape)
        assert np.array_equal(kv_q68.digest(o), gold[tag + item + "o"]), "unpack is not bit-exact"


def test_q8_roundtrip_error_below_q4():
    """Relative L2 of pack -> unpack on N(0, 1) rows.  Measured: Q4 9.4e-2, Q8 6.0e-3 (an 8-bit step is 1/16 of a 4-bit one)."""
    x = np.random.default_rng(5).normal(0, 1, size=(64, 1024)).astype(np.float16)
    e4 = oracle.rel_l2(oracle.kv_unpack_q4(*oracle.kv_pack_q4(x)).astype(np.float64), x.astype(np.float64))
    e8 = oracle.rel_l2(kv_q68.kv_unpack_q8(*kv_q68.kv_pack_q8(x)).astype(np.float64), x.astype(np.float64))
    assert 0.05 < e4 < 0.12
    assert e8 < 8e-3 and e8 < e4 / 10


def test_q8_pack_layout_and_zero_block():
    """An all-zero 64-value unit packs to scale 0 and bytes 0 (0 / 0 = NaN -> 0, as __half2int_rn does) and unpacks to zeros;
    the unit beside it is unaffected."""
    x = np.zeros((1, 128), dtype=np.float16)
    x[0, 64:] = np.linspace(-1, 1, 64).astype(np.float16)
    q, s = kv_q68.kv_pack_q8(x)
    assert q.shape == (1, 128) and s.shape == (1, 4)
    assert not q[0, :64].any() and not s[0, :2].astype(np.float32).any()
    assert np.array_equal(kv_q68.kv_unpack_q8(q, s)[0, :64].astype(np.float32), np.zeros(64, dtype=np.float32))
    y = kv_q68.kv_unpack_q8(q, s)[0, 64:].astype(np.float64)
    assert oracle.rel_l2(y, x[0, 64:].astype(np.float64)) < 1e-2


def _sylvester(n):
    h = np.ones((1, 1))
    while h.shape[0] < n:
        h = np.block([[h, h], [h, -h]])
    return h


@pytest.mark.parametrize("bits", [4, 8])
def test_kv_unpack_exact(bits):
    """kv_q68.kv_unpack_exact: per 64-value unit, each of the two interleaved 32-value halves is H32 (Sylvester order) times
    (code - offset) x scale, / 32, in fp64 -- restated here with an explicit matrix -- and it agrees with the oracle's fp16
    dequantisation to that path's roundings."""
    rng = np.random.default_rng(40 + bits)
    x = rng.normal(0, 1, size=(64, 2, 128)).astype(np.float16)
    q, s = kv_q68.kv_pack(x, bits)
    got = kv_q68.kv_unpack_exact(q, s, bits)
    if bits == 8:
        codes = q.astype(np.float64) - 128
    else:
        codes = np.empty(q.shape[:-1] + (q.shape[-1] * 2,))
        codes[..., 0::2], codes[..., 1::2] = q & 0xF, q >> 4
        codes -= 8
    w = (codes * np.repeat(s.astype(np.float64), 32, axis=-1)).reshape(codes.shape[:-1] + (-1, 32, 2))
    want = np.einsum("ij,...jp->...ip", _sylvester(32), w).reshape(codes.shape) / 32
    assert np.array_equal(got, want)
    fp16 = kv_q68.kv_unpack(q, s, bits).astype(np.float64)
    assert np.abs(fp16 - got).max() <= 4e-3 * np.abs(got).max()
    assert not np.array_equal(fp16, got)
