"""Device state the library keeps between calls, checked across calls, CUDA graphs and streams.

  * The split-KV scratch of the fused decode attention (partial results + arrival counters, csrc/attn_q4.cu attn_scratch)
    is per (device, stream), sized at its bound once, and never moves: a graph captured on a stream keeps valid pointers
    however large the later launches on it or on other streams are; two decoders (a draft model beside a main model) can
    each replay their captured step; launches on two streams at once never merge each other's partial results.
  * The RMSNorm weight of a bare single-row norm + GEMV call (gemv_norm, the decode head) is read as it is at that call:
    updated in place, freed and re-allocated at the same address, alternated, or changed between a capture and its replay.

Every attention output is compared with its serial (or eager) bits and, once per shape, with fp64 attention over the
oracle-dequantised cache (tests/attn_regimes.py) within test_gpu_attn_regimes.py's tolerance; every head output with the
fp64 product rms_norm(x, w) @ W over the library's reconstruct(), within test_gpu_row_blocks.py's 1e-3.
Graphs are replayed one at a time on one stream (DESIGN.md §4: concurrent replays are not supported)."""
import numpy as np
import pytest
import torch

import attn_regimes as ar
import exl2_oracle as oracle

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ATTN_TOL = dict(rel=1.6e-3, mx=2.5e-3)        # test_gpu_attn_regimes.TOL
GEMV_TOL = 1e-3                                # test_gpu_row_blocks.TOL


# ---- fused decode attention ---------------------------------------------------------------------------------------------

def sms() -> int:
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def attn_case(wbits, H, KVH, B, hd, max_ctx, seqlens, seed):
    """A random paged cache, one query row per sequence and its new K/V rows, on the device and as numpy."""
    kb, vb = ar.widths(wbits)
    rng = np.random.default_rng(seed)
    pps = max_ctx // ar.PAGE
    bt = rng.permutation(B * pps).reshape(B, pps).astype(np.int32)
    shp = (B * pps, ar.PAGE, KVH)
    c = dict(wbits=wbits, kb=kb, vb=vb, H=H, KVH=KVH, B=B, hd=hd, max_ctx=max_ctx, seqlens=list(seqlens), bt=bt,
             sigma=1.0 / np.sqrt(hd),
             kq=rng.integers(0, 256, size=shp + (hd * kb // 8,), dtype=np.uint8),
             vq=rng.integers(0, 256, size=shp + (hd * vb // 8,), dtype=np.uint8),
             ks=(rng.uniform(0.05, 0.15, size=shp + (hd // 32,)) / (16 if kb == 8 else 1)).astype(np.float16),
             vs=(rng.uniform(0.02, 0.3, size=shp + (hd // 32,)) / (16 if vb == 8 else 1)).astype(np.float16),
             q=rng.normal(0, 4, size=(B, 1, H, hd)).astype(np.float16),
             kn=rng.normal(0, 1, size=(B, 1, KVH, hd)).astype(np.float16),
             vn=rng.normal(0, 1, size=(B, 1, KVH, hd)).astype(np.float16))
    c["dev"] = {k: torch.from_numpy(np.ascontiguousarray(c[k])).to(DEV) for k in ("kq", "vq", "ks", "vs", "q", "kn", "vn", "bt")}
    c["dev"]["seqlens"] = torch.tensor(c["seqlens"], dtype=torch.int32, device=DEV)
    return c


def launch(c, out):
    """One attention launch on the current stream.  The kernel appends the same new rows to the same slots every time (the
    cache lengths are not advanced), so repeated launches read the same inputs."""
    from exllamav2_b200 import ext as ext_c
    d = c["dev"]
    ext_c.paged_attn_decode_q4(d["q"], d["kn"], d["vn"], d["kq"], d["ks"], d["vq"], d["vs"], d["seqlens"], d["bt"], out, c["sigma"],
                               wbits=c["wbits"])


def new_out(c):
    return torch.zeros((c["B"], 1, c["H"], c["hd"]), dtype=torch.half, device=DEV)


def check_truth(c, out):
    K = [ar.gather_rows(c["kq"], c["ks"], c["bt"], b, sl, c["kb"]) for b, sl in enumerate(c["seqlens"])]
    V = [ar.gather_rows(c["vq"], c["vs"], c["bt"], b, sl, c["vb"]) for b, sl in enumerate(c["seqlens"])]
    truth = ar.attention_truth(c["q"], c["kn"], c["vn"], K, V, c["seqlens"], c["sigma"])
    g = out.cpu().numpy().astype(np.float64)
    assert np.isfinite(g).all()
    rel = np.linalg.norm(g - truth, axis=-1) / np.maximum(np.linalg.norm(truth, axis=-1), 1e-30)
    mx = np.abs(g - truth).max(-1) / np.maximum(np.abs(truth).max(-1), 1e-30)
    assert rel.max() <= ATTN_TOL["rel"] and mx.max() <= ATTN_TOL["mx"], (rel.max(), mx.max())


def same_bits(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


def scratch(stream):
    from exllamav2_b200 import ext as ext_c
    return ext_c.debug_scratch(DEV, stream, "attn_ws"), ext_c.debug_scratch(DEV, stream, "attn_cnt")


def test_split_scratch_survives_larger_launches():
    """A launch with a small split (H 4, B 1, 2048 positions: 4 chunks) is captured on stream s.  Launches that need far more
    split scratch -- H 32 x B 4 at 4096 positions, hd 64 and hd 128 -- then run eagerly on s and on the default stream; s's
    scratch must keep its address and size through all of them (checked after each, before anything could write through a
    moved pointer).  Only then is the graph replayed: bit for bit a fresh eager launch, and within tolerance of fp64."""
    from exllamav2_b200 import ext as ext_c
    small = attn_case(4, 4, 4, 1, 64, 2048, [2000], seed=1)
    assert ar.nsplit_of(1, 2048, 4, 1, sms()) == 4
    s = torch.cuda.Stream(DEV)
    out_g = new_out(small)
    with torch.cuda.stream(s):
        launch(small, out_g)                  # first split launch on s: creates its scratch outside the capture
    torch.cuda.synchronize()
    pinned = scratch(s)
    (ws, ws_bytes), (cnt, cnt_bytes) = pinned
    assert ws and cnt and ws_bytes >= 4 * 4 * 66 * 4 and cnt_bytes >= 4 * 4
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        launch(small, out_g)
    torch.cuda.synchronize()
    big = [attn_case(4, 32, 8, 4, hd, 4096, [4095, 3000, 2100, 1025], seed=2 + hd) for hd in (64, 128)]
    for c in big:
        assert ar.nsplit_of(1, 4096, 32, 4, sms()) == 2
        need = 4 * 32 * 2 * (c["hd"] + 2) * 4        # bytes: 8x and 16x what the small launch needs (4 * 4 * 66 floats)
        for stream in (s, torch.cuda.default_stream(DEV)):
            out = new_out(c)
            with torch.cuda.stream(stream):
                launch(c, out)
            torch.cuda.synchronize()
            assert scratch(s) == pinned, "stream s's split-KV scratch moved under its captured graph"
            d_ws = scratch(stream)[0]
            assert d_ws[1] >= need
            if stream is not s:
                assert d_ws[0] != ws, "two streams share split-KV scratch"
        check_truth(c, out)
    out_g.zero_()
    with torch.cuda.stream(s):
        g.replay()
    torch.cuda.synchronize()
    assert ext_c.paged_attn_status(DEV) == 0
    out_e = new_out(small)
    launch(small, out_e)
    torch.cuda.synchronize()
    assert same_bits(out_g, out_e), "graph replay differs from an eager launch"
    check_truth(small, out_g)


def test_concurrent_streams_split_kv():
    """Two streams, each with its own cache and split shape: Q4 H 8 B 1 over 16384 positions (ring, 16 chunks) and Q8 H 8
    B 2 over 4096 (8 chunks, two sequences), both at hd 128, enqueued alternately, 20 launches per stream with no
    synchronisation between them.  Every output must equal its serially computed bits: two launches that shared split-KV scratch would write the
    same partial-result slots and bump the same arrival counters.  (42 attention launches in all: fewer than the 127 slot
    counters of the per-device ring, so no two launches in flight share one.)"""
    from exllamav2_b200 import ext as ext_c
    c1 = attn_case(4, 8, 8, 1, 128, 16384, [16383], seed=7)
    c2 = attn_case(8, 8, 2, 2, 128, 4096, [4095, 3000], seed=8)
    p1 = ar.plan(4, 128, 8, 1, 1, 16384, c1["seqlens"], sms())
    p2 = ar.plan(8, 128, 8, 2, 1, 4096, c2["seqlens"], sms())
    # each launch takes one CTA slot per SM (slot holders pad its grid to the SM count), with ~90 KB of shared memory at hd 128:
    # one CTA of each fits on an SM together.  (A launch of much smaller shared memory runs under another shared-memory
    # configuration of the SM and does not share one with these.)
    assert p1["smem"] + p2["smem"] <= 200 * 1024
    assert p1["nsplit"] == 16 and {"ring", "merge"} <= ar.branches(p1, 1, 8, 1, sms())
    assert p2["nsplit"] == 8 and "merge_batch" in ar.branches(p2, 1, 8, 2, sms())
    s1, s2 = torch.cuda.Stream(DEV), torch.cuda.Stream(DEV)
    want1, want2 = new_out(c1), new_out(c2)
    with torch.cuda.stream(s1):
        launch(c1, want1)
    torch.cuda.synchronize()
    with torch.cuda.stream(s2):
        launch(c2, want2)
    torch.cuda.synchronize()
    check_truth(c1, want1)
    check_truth(c2, want2)
    outs1 = [new_out(c1) for _ in range(20)]
    outs2 = [new_out(c2) for _ in range(20)]
    torch.cuda.synchronize()
    # Both streams are held for ~20 ms, so that all 40 launches are queued before the first one runs, rather than issued one
    # at a time as the host gets to them.  A plain kernel follows every attention launch: it keeps the stream's next launch
    # from being started early (programmatic dependent launch), which would fill each SM's second CTA slot with the same
    # stream's work.  So each stream has one launch on the GPU at a time, and the two streams' launches share every SM.
    for s in (s1, s2):
        with torch.cuda.stream(s):
            torch.cuda._sleep(40_000_000)
    for o1, o2 in zip(outs1, outs2):
        for s, c, o in ((s1, c1, o1), (s2, c2, o2)):
            with torch.cuda.stream(s):
                launch(c, o)
                torch.cuda._sleep(1000)
    torch.cuda.synchronize()
    assert ext_c.paged_attn_status(DEV) == 0
    bad1 = [i for i, o in enumerate(outs1) if not same_bits(o, want1)]
    bad2 = [i for i, o in enumerate(outs2) if not same_bits(o, want2)]
    assert not bad1 and not bad2, f"concurrent launches disturbed each other: stream 1 {bad1}, stream 2 {bad2}"


# ---- two decoders in one process ----------------------------------------------------------------------------------------

def _decoder(preset, cache_len):
    from exllamav2_b200.model import PRESETS, ExLlamaV2Decoder
    return ExLlamaV2Decoder(PRESETS[preset](), device=DEV, seed=3, batch_size=1, cache_len=cache_len)


def _logits(dec, ids):
    return dec.decode(ids).clone()


def test_two_decoders_one_process():
    """Decoder A (test-tiny, H 4, 2048 positions: 4 split chunks) captures its step.  Decoder B (test-small, H 8, 4096
    positions: 8 chunks, 4x A's split scratch) prefills, decodes one step eagerly, then captures.  Replays of A and B then
    alternate on one stream.  Every step's logits must equal, bit for bit, those of the same decoder run alone over the
    same tokens (prefill, capture -- B after its eager step --, replays)."""
    assert ar.nsplit_of(1, 2048, 4, 1, sms()) == 4 and ar.nsplit_of(1, 4096, 8, 1, sms()) == 8
    g = torch.Generator().manual_seed(12)
    pa, ga = torch.randint(0, 512, (1, 7), generator=g).to(DEV), torch.randint(0, 512, (1, 6), generator=g).to(DEV)
    pb, gb = torch.randint(0, 512, (1, 9), generator=g).to(DEV), torch.randint(0, 512, (1, 7), generator=g).to(DEV)

    def alone(preset, cache_len, prompt, gen, eager_first):
        dec = _decoder(preset, cache_len)
        assert dec.chained and dec.fused_attn
        dec.prefill(prompt)
        out = []
        if eager_first:
            out.append(_logits(dec, gen[:, :1]))
        dec.capture()
        for t in range(len(out), gen.shape[1]):
            out.append(_logits(dec, gen[:, t:t + 1]))
        torch.cuda.synchronize()
        dec.unload()
        return out

    solo_a = alone("test-tiny", 2048, pa, ga, False)
    solo_b = alone("test-small", 4096, pb, gb, True)
    a = _decoder("test-tiny", 2048)
    a.prefill(pa)
    a.capture()
    b = _decoder("test-small", 4096)
    b.prefill(pb)
    got_b = [_logits(b, gb[:, :1])]
    b.capture()
    got_a = []
    for t in range(ga.shape[1]):
        got_a.append(_logits(a, ga[:, t:t + 1]))
        if t + 1 < gb.shape[1]:
            got_b.append(_logits(b, gb[:, t + 1:t + 2]))
    torch.cuda.synchronize()
    for name, got, want in (("A", got_a, solo_a), ("B", got_b, solo_b)):
        assert len(got) == len(want)
        for t, (x, y) in enumerate(zip(got, want)):
            assert torch.isfinite(x.float()).all()
            assert same_bits(x, y), f"decoder {name}, step {t}: logits differ from the decoder run alone"
    a.unload()
    b.unload()


# ---- the RMSNorm weight of a bare norm + GEMV call ------------------------------------------------------------------------

K_HEAD, N_HEAD, EPS = 1024, 768, 1e-5


@pytest.fixture(scope="module")
def head():
    """An act-order (permuted) 4-bit matrix as the decode head, its fp64 weights, one input row and two norm weights whose
    results differ by far more than the tolerance."""
    from exllamav2_b200 import synthetic
    from exllamav2_b200.linear import ExLlamaV2Linear
    lin = ExLlamaV2Linear(K_HEAD, N_HEAD, device=DEV)
    lin.load(synthetic.random_linear(K_HEAD, N_HEAD, ((4,), (1.0,), 128), device=DEV, seed=31, weight_std=K_HEAD ** -0.5))
    gen = torch.Generator().manual_seed(9)
    W = lin.get_weight_tensor_dq().cpu().numpy().astype(np.float64)
    x = torch.randn((1, K_HEAD), generator=gen).half()
    wa = (1 + 0.1 * torch.randn((K_HEAD,), generator=gen)).half()
    wb = (0.2 + 1.5 * torch.rand((K_HEAD,), generator=gen)).half()
    h = dict(lin=lin, W=W, x=x.to(DEV), wa=wa, wb=wb)
    ta, tb = truth(h, wa), truth(h, wb)
    assert oracle.rel_l2(ta, tb) > 100 * GEMV_TOL
    yield h
    lin.unload()


def truth(h, w_cpu):
    xn = oracle.rms_norm(h["x"].cpu().numpy(), w_cpu.numpy(), EPS)
    return xn.astype(np.float64) @ h["W"]


def head_call(h, w, out=None):
    from exllamav2_b200 import ext as ext_c
    out = torch.empty((1, N_HEAD), dtype=torch.half, device=DEV) if out is None else out
    ext_c.gemv_norm(h["x"], h["lin"].q_handle, w, EPS, out)
    return out


def check_head(h, out, w_cpu, what):
    torch.cuda.synchronize()
    err = oracle.rel_l2(out.cpu().numpy().astype(np.float64), truth(h, w_cpu))
    assert err <= GEMV_TOL, f"{what}: rel_l2 {err:.2e} against rms_norm(x, w) @ W"


def test_norm_weight_updated_in_place(head):
    w = head["wa"].to(DEV)
    check_head(head, head_call(head, w), head["wa"], "first weight")
    w.copy_(head["wb"].to(DEV))
    check_head(head, head_call(head, w), head["wb"], "same tensor after copy_")


def test_norm_weight_reallocated_at_same_address(head):
    w = head["wa"].to(DEV)
    check_head(head, head_call(head, w), head["wa"], "first weight")
    addr = w.data_ptr()
    del w
    w2 = torch.empty((K_HEAD,), dtype=torch.half, device=DEV)
    if w2.data_ptr() != addr:
        pytest.skip("the caching allocator did not hand the freed block back")
    w2.copy_(head["wb"])
    check_head(head, head_call(head, w2), head["wb"], "new weight at the freed address")


def test_norm_weights_alternate(head):
    wa, wb = head["wa"].to(DEV), head["wb"].to(DEV)
    for w, w_cpu, what in ((wa, head["wa"], "A"), (wb, head["wb"], "B"), (wa, head["wa"], "A again")):
        check_head(head, head_call(head, w), w_cpu, what)


def test_norm_weight_graph_keeps_its_weight(head):
    """A graph captured with weight A, then an eager call with weight B, then the replay: the replay must give A's result,
    bit for bit the eager call with A."""
    wa, wb = head["wa"].to(DEV), head["wb"].to(DEV)
    s = torch.cuda.Stream(DEV)
    out_g = torch.empty((1, N_HEAD), dtype=torch.half, device=DEV)
    with torch.cuda.stream(s):
        head_call(head, wa, out_g)                # first launch of this structure (plans) outside the capture
    torch.cuda.synchronize()
    want = out_g.clone()
    check_head(head, want, head["wa"], "eager A")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        head_call(head, wa, out_g)
    check_head(head, head_call(head, wb), head["wb"], "eager B between capture and replay")
    out_g.zero_()
    with torch.cuda.stream(s):
        g.replay()
    torch.cuda.synchronize()
    assert same_bits(out_g, want), "the replay did not keep the weight it was captured with"
