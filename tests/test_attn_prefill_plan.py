"""CPU: the prompt attention's launch arithmetic (tests/attn_prefill_plan.py) against the library and DESIGN.md §3.8.

The library checks every argument before its first CUDA call, so its shared-memory refusal is probed here without a GPU: a page
table one entry past attn_prefill_plan.max_pages() is refused with the byte count the plan computes, and the largest accepted
one gets past that check to the next refusal (batch 0), never to a launch."""
import ctypes

import pytest

import attn_prefill_plan as ap


@pytest.fixture(scope="module")
def lib():
    from exllamav2_b200 import ext
    return ext.lib


def _call(lib, wbits=4, hd=128, H=8, KVH=2, batch=1, q_len=1, page_size=256, pps=1):
    fake = ctypes.c_void_p(0x1000)          # never dereferenced: every call below is refused before any CUDA call
    rc = lib.exl2b_paged_attn_prefill_q(*([fake] * 10), batch, q_len, H, KVH, hd, page_size, pps, 0.1, wbits, None)
    return rc, lib.exl2b_last_error().decode()


def test_shared_memory_map_figures():
    """The figures DESIGN.md §3.8 states: a CTA's bytes at a 16-page table (4096 positions), per format and head dim."""
    want = {(4, 64): 36928, (6, 64): 41024, (8, 64): 45120, (4, 128): 71744, (6, 128): 79936, (8, 128): 88128}
    got = {k: ap.smem_bytes(*k, 16)["total"] for k in want}
    assert got == want
    for (w, hd) in want:
        s = ap.smem_bytes(w, hd, 16)
        assert s["out"] <= s["tiles"]          # the fp32 output tile fits over the fp16 operand tiles it replaces
        assert 2 * s["total"] <= 228 * 1024    # two CTAs per SM at the decoder's cache lengths


@pytest.mark.parametrize("wbits,hd", [(4, 64), (6, 64), (8, 64), (4, 128), (6, 128), (8, 128)])
def test_largest_page_table_and_one_more_is_refused(lib, wbits, hd):
    n = ap.max_pages(wbits, hd)
    assert ap.smem_bytes(wbits, hd, n)["fits"] and not ap.smem_bytes(wbits, hd, n + 1)["fits"]
    rc, msg = _call(lib, wbits, hd, pps=n + 1)
    assert rc != 0 and "shared memory" in msg and f"{ap.smem_bytes(wbits, hd, n + 1)['total']} bytes" in msg, msg
    rc, msg = _call(lib, wbits, hd, pps=n, batch=0)
    assert rc != 0 and "bad shape" in msg, msg


@pytest.mark.parametrize("kw,words", [
    (dict(wbits=5), "wbits"), (dict(hd=96), "head_dim 96"), (dict(H=6, KVH=4), "GQA ratio"),
    (dict(page_size=96), "page_size 96"), (dict(q_len=0), "bad shape"),
])
def test_argument_refusals(lib, kw, words):
    rc, msg = _call(lib, **kw)
    assert rc != 0 and words in msg, msg


def test_grid_and_append_ownership():
    """Every new token is appended by exactly one CTA, and the key tiles of a CTA end at its last query's position."""
    for q_len in (1, 9, 63, 64, 65, 200, 2048):
        for group in (1, 4, 7, 8):
            nmb = ap.grid(q_len, 4 * group, 4, 1)[0]
            owners = [t for mb in range(nmb) for t in ap.appended_tokens(mb, q_len, group)]
            assert owners == list(range(q_len))
            for seqlen in (0, 255, 4095):
                last = ap.key_tiles(seqlen, nmb - 1, q_len, group)
                assert last == (seqlen + q_len + ap.AP_BN - 1) // ap.AP_BN
                assert all(ap.key_tiles(seqlen, mb, q_len, group) <= last for mb in range(nmb))
    assert ap.grid(2048, 8, 2, 1) == (128, 2, 1) and ap.grid(65, 28, 4, 3) == (8, 4, 3)
