"""The batch-1 GEMV (csrc/gemv_i8.cu) with its group scales and stage lists fed through shared memory, on the structures
that exercise that plumbing: a fused launch whose warps change matrix, GPTQ's 128-byte scale | zero rows, every stage
flushing with the scale ring wrapping, a group spanning two stages, a ragged last column block, stage lists longer than the
list window, and CUDA graph replays.  Each result is checked against the fp64 product with the library's reconstruct()
weights (<= 5e-4 relative L2), and a unit-vector row must return those fp16 weights bit for bit."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 5e-4


def _lin(K, N, plan, seed, perm_seed=None):
    from exllamav2_b200 import synthetic
    from exllamav2_b200.linear import ExLlamaV2Linear
    w = synthetic.random_linear(K, N, plan, device=DEV, seed=seed, weight_std=1.0 / math.sqrt(K), perm_seed=perm_seed)
    lin = ExLlamaV2Linear(K, N, device=DEV)
    lin.load(w)
    return lin


def _rel(got: torch.Tensor, want: torch.Tensor) -> float:
    return (torch.linalg.norm(got.double() - want) / torch.linalg.norm(want)).item()


def _row(K, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn((1, K), device=DEV, generator=g).half()


def _gemv(lin, x, N):
    from exllamav2_b200 import ext as ext_c
    c = torch.empty((1, N), dtype=torch.half, device=DEV)
    ext_c.gemm_half_q_half(x, lin.q_handle, c)
    return c


def _check_linear(lin, K, N, seed=0):
    W = lin.get_weight_tensor_dq()
    assert W.shape == (K, N)
    x = _row(K, seed)
    err = _rel(_gemv(lin, x, N), x.double() @ W.double())
    assert err <= TOL, f"rel_l2 {err:.2e}"
    # unit-vector rows: the fp16 weights themselves (exact row quantisation, exact integer sums, one rounding)
    for k in (0, K // 3, K - 1):
        e = torch.zeros((1, K), dtype=torch.half, device=DEV)
        e[0, k] = 1.0
        got = _gemv(lin, e, N)
        assert torch.equal(got[0].view(torch.int16), W[k].view(torch.int16)), f"unit row {k} differs from reconstruct()"


CASES = {
    # GPTQ g128 with act-order: 128-byte scale | zero rows
    "gptq_g128_act": (4096, 1024, ("gptq", 128, True)),
    # 8-bit g32 then 2-bit g64: every stage flushes, the scale ring wraps many times
    "b8_g32_b2_g64": (2048, 512, ((8, 2), (0.25, 0.75), (32, 64))),
    # g256: a group spans two stages, only the second flushes
    "b4_g256": (2048, 1024, ((4,), (1.0,), 256)),
    # N = 1000: the last column block is ragged (its scale row reads into the table's padding)
    "n1000_ragged": (1024, 1000, ((4, 3), (0.5, 0.5), 128)),
    # K = 16384, N = 4096, 8-bit g32: 32 one-slab stages per warp, twice the list window (test_i8_smem_operands.py checks
    # the plan of this structure)
    "long_lists": (16384, 4096, ((8,), (1.0,), 32)),
}


@pytest.mark.parametrize("name", list(CASES))
def test_gemv_smem_operands(name):
    K, N, plan = CASES[name]
    lin = _lin(K, N, plan, seed=sum(map(ord, name)))
    _check_linear(lin, K, N)
    lin.unload()


def test_fused_qkv_54():
    """Q|K|V [5,4] in one launch with the RMSNorm prologue: warps whose range crosses from one matrix into the next."""
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200.ext import none_tensor
    hid, H, hd = 4096, 32, 128
    m54 = ((5, 4), (0.1, 0.9), 128)
    lq, lk, lv = _lin(hid, hid, m54, 41, 41), _lin(hid, 1024, m54, 42, 41), _lin(hid, 1024, m54, 43, 41)
    lo = _lin(hid, hid, m54, 44)
    g = torch.Generator(device=DEV).manual_seed(5)
    nw = (1 + 0.1 * torch.randn((hid,), device=DEV, generator=g)).half()
    hat = ext_c.make_q_attn(nw, none_tensor, True, False, 1e-5, lq.q_handle, lk.q_handle, lv.q_handle, lo.q_handle,
                            none_tensor, none_tensor, 64, hid, H, 8, hd, 64, True, 2, hd,
                            none_tensor, none_tensor, none_tensor, none_tensor, False, True)
    x = torch.randn((1, 1, hid), device=DEV, generator=g).half()
    q = torch.empty((1, 1, hid), dtype=torch.half, device=DEV)
    k, v = (torch.empty((1, 1, 1024), dtype=torch.half, device=DEV) for _ in range(2))
    ext_c.q_attn_forward_1(hat, x, 1, 1, 0, none_tensor, q, k, v, none_tensor, none_tensor)
    xf = x[0].double()
    xn = xf * nw.double() / torch.sqrt((xf * xf).mean(-1, keepdim=True) + 1e-5)
    for nm, got, lin in (("q", q, lq), ("k", k, lk), ("v", v, lv)):
        err = _rel(got[0], xn @ lin.get_weight_tensor_dq().double())
        assert err <= TOL, f"{nm}: rel_l2 {err:.2e}"
    ext_c.free_q_attn(hat)
    for l in (lq, lk, lv, lo):
        l.unload()


def test_graph_replays_bit_identical():
    from exllamav2_b200 import ext as ext_c
    K, N = 4096, 11008
    lin = _lin(K, N, ((5, 4), (0.1, 0.9), 128), 51)
    x = _row(K, 6)
    c = torch.empty((1, N), dtype=torch.half, device=DEV)
    s = torch.cuda.Stream(DEV)
    with torch.cuda.stream(s):
        ext_c.gemm_half_q_half(x, lin.q_handle, c)           # plans the launch structure outside the capture
        torch.cuda.synchronize()
        eager = c.clone()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            ext_c.gemm_half_q_half(x, lin.q_handle, c)
    outs = []
    for _ in range(2):
        c.zero_()
        graph.replay()
        torch.cuda.synchronize()
        outs.append(c.clone())
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16)), "two replays differ"
    assert torch.equal(outs[0].view(torch.int16), eager.view(torch.int16)), "replay differs from the eager launch"
    assert _rel(outs[0][0], x[0].double() @ lin.get_weight_tensor_dq().double()) <= TOL
    del graph
    lin.unload()
