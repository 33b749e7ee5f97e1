"""GPU parity tests of the quantized-linear path, through the C ABI (ctypes) against the CPU oracle.

Modelled on the reference's tests/test_gemv.py: quantized forward vs reconstruct+matmul, identity-matrix input
("ident" must be bit-exact), random-input error -- but with asserts and explicit tolerances:
  * reconstruct: BIT-EXACT vs oracle (integer unpack indexing + one fp16 multiply)
  * gemm: rel-L2 vs fp64 truth <= 5e-4 (fp32 accumulate + one fp16 rounding of the output; the reference's own
    fp16-accumulating kernel sits near 1e-3, north_star tolerance is 1e-3)
"""
import numpy as np
import pytest
import torch

import cases
import exl2_oracle as oracle

pytestmark = pytest.mark.gpu

GEMM_TOL = 5e-4
DEV = "cuda:0"


def _load(name):
    from exllamav2_b200.linear import ExLlamaV2Linear, load_tensor_dict
    w_np = cases.make_case(name)
    K, N = cases.case_shape(name)
    lin = ExLlamaV2Linear(K, N, has_bias="bias" in w_np, key=name, device=DEV)
    lin.load(load_tensor_dict(w_np, DEV))
    return lin, w_np


def _oracle_w(name, w_np):
    return oracle.exl2_reconstruct(w_np) if name in cases.EXL2_CASES else oracle.gptq_reconstruct(w_np)


ALL = list(cases.EXL2_CASES) + list(cases.GPTQ_CASES)


@pytest.mark.parametrize("name", ALL)
def test_reconstruct_bit_exact(name):
    lin, w_np = _load(name)
    got = lin.get_weight_tensor_dq().cpu().numpy()
    want = _oracle_w(name, w_np)
    assert got.shape == want.shape
    assert np.array_equal(cases.u16(got), cases.u16(want)), f"{name}: {np.count_nonzero(cases.u16(got) != cases.u16(want))} mismatching weights"
    lin.unload()


@pytest.mark.parametrize("name", ALL)
def test_identity_input_equals_reconstruct(name):
    """tests/test_gemv.py:155-159 'ident': forward(I) must reproduce reconstruct() exactly (+ bias)."""
    lin, w_np = _load(name)
    K, N = cases.case_shape(name)
    eye = torch.eye(K, dtype=torch.half, device=DEV)
    got = lin.forward(eye).float().cpu().numpy()
    want = _oracle_w(name, w_np).astype(np.float32)
    if "bias" in w_np:
        want = (want + w_np["bias"].astype(np.float32)).astype(np.float16).astype(np.float32)
        assert np.allclose(got, want, atol=2e-3, rtol=2e-3)
    else:
        assert np.array_equal(got, want), f"{name}: {np.count_nonzero(got != want)} mismatches"
    lin.unload()


@pytest.mark.parametrize("name", ALL)
@pytest.mark.parametrize("M", cases.M_VALUES)
def test_gemm_vs_truth(name, M):
    lin, w_np = _load(name)
    a = cases.activations(name, M)
    truth = oracle.gemm_truth(a, _oracle_w(name, w_np), w_np.get("bias"))
    got = lin.forward(torch.from_numpy(a).to(DEV)).cpu().numpy()
    err = oracle.rel_l2(got, truth)
    assert err <= GEMM_TOL, f"{name} M={M}: rel_l2 {err:.2e}"
    lin.unload()


@pytest.mark.parametrize("name", ["b4_g128", "b54_g64", "gptq_g128_act", "b4_n96_ragged"])
def test_gemm_accumulate_and_strided(name):
    """clear=false form (residual add) and non-contiguous row strides."""
    from exllamav2_b200 import ext as ext_c
    lin, w_np = _load(name)
    K, N = cases.case_shape(name)
    a = cases.activations(name, 3)
    c0 = np.random.default_rng(5).normal(0, 1, size=(3, N)).astype(np.float16)
    a_buf = torch.zeros((3, K + 24), dtype=torch.half, device=DEV)
    a_buf[:, :K] = torch.from_numpy(a).to(DEV)
    c_buf = torch.zeros((3, N + 8), dtype=torch.half, device=DEV)
    c_buf[:, :N] = torch.from_numpy(c0).to(DEV)
    ext_c.gemm_half_q_half_accum(a_buf[:, :K], lin.q_handle, c_buf[:, :N])
    truth = oracle.gemm_truth(a, _oracle_w(name, w_np), w_np.get("bias"), c0)
    assert oracle.rel_l2(c_buf[:, :N].cpu().numpy(), truth) <= GEMM_TOL
    assert torch.count_nonzero(c_buf[:, N:]).item() == 0
    lin.unload()


def test_gptq_v2_zero_offset():
    """gptq_v2 checkpoints: qzeros -= 0x11111111 before use (ext.py:366-367)."""
    from exllamav2_b200.linear import ExLlamaV2Linear, load_tensor_dict
    w_np = cases.make_case("gptq_g128")
    # keep nibbles >= 1 so the subtraction does not borrow across nibbles
    qz = w_np["qzeros"].view(np.uint32) | np.uint32(0x11111111)
    w_np["qzeros"] = qz.view(np.int32)
    want = oracle.gptq_reconstruct(w_np, offset_qzeros=True)
    lin = ExLlamaV2Linear(256, 128, device=DEV)
    lin.load(load_tensor_dict(w_np, DEV), offset_qzeros=True)
    assert np.array_equal(cases.u16(lin.get_weight_tensor_dq().cpu().numpy()), cases.u16(want))
    lin.unload()


def test_prescale_folds_into_scale_max():
    from exllamav2_b200.linear import ExLlamaV2Linear, load_tensor_dict
    w_np = cases.make_case("b4_g128")
    want = oracle.exl2_reconstruct(w_np, prescale=0.5)
    lin = ExLlamaV2Linear(256, 128, prescale=0.5, device=DEV)
    lin.load(load_tensor_dict(w_np, DEV))
    assert np.array_equal(cases.u16(lin.get_weight_tensor_dq().cpu().numpy()), cases.u16(want))
    lin.unload()


def test_error_behaviour():
    from exllamav2_b200 import ext as ext_c
    lin, _ = _load("b4_g128")
    a = torch.zeros((1, 128), dtype=torch.half, device=DEV)      # wrong K
    c = torch.zeros((1, 128), dtype=torch.half, device=DEV)
    with pytest.raises(RuntimeError, match="incompatible shapes"):
        ext_c.gemm_half_q_half(a, lin.q_handle, c, False)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ext_c.gemm_half_q_half(torch.zeros((1, 256), dtype=torch.half), lin.q_handle, c, False)
    with pytest.raises(RuntimeError, match="datatype"):
        ext_c.gemm_half_q_half(torch.zeros((1, 256), dtype=torch.float, device=DEV), lin.q_handle, c, False)
    lin.unload()


# ---- BASELINE.json full sizes: size-independent properties ------------------------------------------------------

FULL = [
    ("llama7b_qkvo", dict(K=4096, N=4096, bits=(4,), bits_prop=(1.0,), group_size=128, seed=101)),
    ("llama7b_gate_54", dict(K=4096, N=11008, bits=(5, 4), bits_prop=(0.1, 0.9), group_size=128, seed=102)),
    ("llama7b_down_43", dict(K=11008, N=4096, bits=(4, 3), bits_prop=(0.1, 0.9), group_size=128, seed=103)),
    ("llama7b_head_6", dict(K=4096, N=32000, bits=(6,), bits_prop=(1.0,), group_size=128, seed=104)),
    ("tinyllama_kv", dict(K=2048, N=256, bits=(4,), bits_prop=(1.0,), group_size=128, seed=105)),
]


@pytest.mark.parametrize("name,kw", FULL, ids=[f[0] for f in FULL])
def test_full_size_properties(name, kw):
    """At full size the numpy oracle is too slow, so check properties that do not need it:
      (1) unit-vector inputs return rows of reconstruct() bit-exactly (unpack indexing at every k, n)
      (2) the kernel agrees with an fp32 matmul over its own reconstruct() output
      (3) linearity: f(a1) + f(a2) ~= f(a1 + a2)   (4) determinism: two runs are bit-identical."""
    import synth
    from exllamav2_b200.linear import ExLlamaV2Linear, load_tensor_dict
    w_np = synth.make_exl2(**kw)
    K, N = kw["K"], kw["N"]
    lin = ExLlamaV2Linear(K, N, device=DEV)
    lin.load(load_tensor_dict(w_np, DEV))
    W = lin.get_weight_tensor_dq()
    rng = np.random.default_rng(kw["seed"])
    rows = rng.choice(K, size=8, replace=False)
    e = torch.zeros((8, K), dtype=torch.half, device=DEV)
    e[torch.arange(8), torch.from_numpy(rows).to(DEV)] = 1.0
    got = lin.forward(e)
    assert torch.equal(got, W[torch.from_numpy(rows).to(DEV)]), "unit-vector rows differ from reconstruct"
    for M in (1, 4, 8):
        a = torch.from_numpy(rng.normal(0, 1, size=(M, K)).astype(np.float16)).to(DEV)
        y = lin.forward(a)
        y2 = lin.forward(a)
        assert torch.equal(y, y2), "non-deterministic output"
        ref = a.float() @ W.float()
        err = (torch.linalg.norm(y.float() - ref) / torch.linalg.norm(ref)).item()
        assert err <= GEMM_TOL, f"{name} M={M}: rel_l2 {err:.2e}"
    a1 = torch.from_numpy(rng.normal(0, 1, size=(1, K)).astype(np.float16)).to(DEV)
    a2 = torch.from_numpy(rng.normal(0, 1, size=(1, K)).astype(np.float16)).to(DEV)
    s = (lin.forward(a1).float() + lin.forward(a2).float())
    t = lin.forward((a1.float() + a2.float()).half()).float()
    assert (torch.linalg.norm(s - t) / torch.linalg.norm(t)).item() <= 2e-3
    lin.unload()


# ---- many rows (prefill): reconstruct + tensor-core GEMM, the reference's regime above MAX_Q_GEMM_ROWS (q_gemm.cu:233-266) ------

@pytest.mark.parametrize("name", ["b4_g128", "b54_g64", "b865_mixed", "b6_g128_bias", "b4_n96_ragged", "gptq_g128_act", "gptq_g64_act_b", "gptq_g32"])
@pytest.mark.parametrize("M", [17, 32, 33, 64, 256])
def test_gemm_many_rows(name, M):
    lin, w_np = _load(name)
    a = cases.activations(name, M)
    truth = oracle.gemm_truth(a, _oracle_w(name, w_np), w_np.get("bias"))
    got = lin.forward(torch.from_numpy(a).to(DEV)).cpu().numpy()
    err = oracle.rel_l2(got, truth)
    assert err <= GEMM_TOL, f"{name} M={M}: rel_l2 {err:.2e}"
    lin.unload()


def test_gemm_many_rows_accumulate_strided():
    from exllamav2_b200 import ext as ext_c
    name = "b6_g128_bias"
    lin, w_np = _load(name)
    K, N = cases.case_shape(name)
    M = 40
    a = cases.activations(name, M)
    c0 = np.random.default_rng(6).normal(0, 1, size=(M, N)).astype(np.float16)
    a_buf = torch.zeros((M, K + 8), dtype=torch.half, device=DEV)
    a_buf[:, :K] = torch.from_numpy(a).to(DEV)
    c_buf = torch.zeros((M, N + 16), dtype=torch.half, device=DEV)
    c_buf[:, :N] = torch.from_numpy(c0).to(DEV)
    ext_c.gemm_half_q_half_accum(a_buf[:, :K], lin.q_handle, c_buf[:, :N])
    truth = oracle.gemm_truth(a, _oracle_w(name, w_np), w_np.get("bias"), c0)
    assert oracle.rel_l2(c_buf[:, :N].cpu().numpy(), truth) <= GEMM_TOL
    assert torch.count_nonzero(c_buf[:, N:]).item() == 0
    lin.unload()


def test_prefill_2048_rows_llama_shape():
    """BASELINE config 3 'bs=16 prefill': 2048 rows through a 4096 x 4096 [5,4] matrix in ONE weight pass; checked against an
    fp32 matmul over the kernel's own (bit-exact) reconstruct."""
    import math
    from exllamav2_b200 import synthetic
    from exllamav2_b200.linear import ExLlamaV2Linear
    w = synthetic.random_exl2(4096, 4096, (5, 4), (0.1, 0.9), 128, device=DEV, seed=9, weight_std=1.0 / math.sqrt(4096))
    lin = ExLlamaV2Linear(4096, 4096, device=DEV)
    lin.load(w)
    a = torch.randn((2048, 4096), device=DEV, generator=torch.Generator(device=DEV).manual_seed(1)).half()
    y = lin.forward(a)
    ref = a.float() @ lin.get_weight_tensor_dq().float()
    err = (torch.linalg.norm(y.float() - ref) / torch.linalg.norm(ref)).item()
    assert err <= GEMM_TOL, f"rel_l2 {err:.2e}"
    lin.unload()


# ---- many rows over more than one column window: gemm_big dequantises at most BIG_TEMP_BYTES of columns at a time ----------

BIG_TEMP_BYTES = 64 << 20       # csrc/gemm_big.cu
STRIP_N = 128                   # columns per strip of the default (tensor-core) layout, csrc/layout.h strip_n
WINDOW_CASES = {                # dequantised 4096 x N fp16 > 64 MB, last strip ragged
    "exl2_54": dict(K=4096, N=8224, bits=(5, 4), bits_prop=(0.1, 0.9), group_size=128, seed=201, bias=True),
    "gptq_act": dict(K=4096, N=8200, group_size=128, seed=202, act_order=True, bias=True),
}
_WINDOW_W = {}


def _windows(K, N):
    """(windows, columns of the last window) of gemm_big_launch for a K x N matrix."""
    per_window = max(1, BIG_TEMP_BYTES // (K * STRIP_N * 2))
    strips = -(-N // STRIP_N)
    n = -(-strips // per_window)
    return n, N - (n - 1) * per_window * STRIP_N


def _window_case(name):
    """(checkpoint tensors incl. bias, oracle W) -- bias is drawn last, so the weights are the same with and without it."""
    import synth
    if name not in _WINDOW_W:
        kw = WINDOW_CASES[name]
        w_np = synth.make_exl2(**kw) if "bits" in kw else synth.make_gptq(**kw)
        W = oracle.exl2_reconstruct(w_np) if "bits" in kw else oracle.gptq_reconstruct(w_np)
        _WINDOW_W[name] = (w_np, W)
    return _WINDOW_W[name]


@pytest.mark.parametrize("M", [17, 40, 300])
@pytest.mark.parametrize("mode", ["clear", "accumulate"])
@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("name", list(WINDOW_CASES))
def test_gemm_many_rows_multi_window(name, bias, mode, M):
    """Every column window after the first (strip0 > 0), the ragged last window, bias and accumulate per window, into a strided
    c whose padding must stay zero -- against fp64 a @ W_oracle."""
    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200.linear import ExLlamaV2Linear, load_tensor_dict
    K, N = WINDOW_CASES[name]["K"], WINDOW_CASES[name]["N"]
    windows, last = _windows(K, N)
    assert windows == 2 and 0 < last < STRIP_N, (windows, last)
    w_full, W = _window_case(name)
    w_np = {k: v for k, v in w_full.items() if bias or k != "bias"}
    lin = ExLlamaV2Linear(K, N, has_bias=bias, key=name, device=DEV)
    lin.load(load_tensor_dict(w_np, DEV))
    rng = np.random.default_rng(M + 7 * bias)
    a = rng.normal(0, 1, size=(M, K)).astype(np.float16)
    c0 = rng.normal(0, 1, size=(M, N)).astype(np.float16)
    a_buf = torch.zeros((M, K + 8), dtype=torch.half, device=DEV)
    a_buf[:, :K] = torch.from_numpy(a).to(DEV)
    c_buf = torch.zeros((M, N + 24), dtype=torch.half, device=DEV)
    c_buf[:, :N] = torch.from_numpy(c0).to(DEV)         # clear: must be overwritten, not added to
    if mode == "clear":
        ext_c.gemm_half_q_half(a_buf[:, :K], lin.q_handle, c_buf[:, :N], False)
    else:
        ext_c.gemm_half_q_half_accum(a_buf[:, :K], lin.q_handle, c_buf[:, :N])
    truth = oracle.gemm_truth(a, W, w_np.get("bias"), c0 if mode == "accumulate" else None)
    got = c_buf[:, :N].cpu().numpy()
    err = oracle.rel_l2(got, truth)
    assert err <= GEMM_TOL, f"{name} bias={bias} {mode} M={M}: rel_l2 {err:.2e}"
    # every window on its own (a wrong window offset leaves the overall error small when the window is narrow)
    c1 = N - last
    err_last = oracle.rel_l2(got[:, c1:], truth[:, c1:])
    assert err_last <= GEMM_TOL, f"last window ({last} columns): rel_l2 {err_last:.2e}"
    assert oracle.rel_l2(got[:, :c1], truth[:, :c1]) <= GEMM_TOL
    assert torch.count_nonzero(c_buf[:, N:]).item() == 0
    lin.unload()


def test_two_streams_do_not_share_scratch():
    """Calls on different streams of one device run concurrently and must not share scratch (SURVEY.md 8b: re-entrant per handle):
    every row regime (1 row: integer GEMV, 4 rows: wgmma kernel, 40 rows: dense path), two matrices, two streams, many
    interleaved launches; results must equal the serial ones bit for bit."""
    from exllamav2_b200 import ext as ext_c
    lin_a, _ = _load("b54_g64")
    lin_b, _ = _load("b43_g128")
    Ka, Na = cases.case_shape("b54_g64")
    Kb, Nb = cases.case_shape("b43_g128")
    for M in (1, 4, 40):
        xa = torch.from_numpy(cases.activations("b54_g64", M)).to(DEV)
        xb = torch.from_numpy(cases.activations("b43_g128", M)).to(DEV)
        want_a, want_b = lin_a.forward(xa).clone(), lin_b.forward(xb).clone()
        torch.cuda.synchronize()
        s1, s2 = torch.cuda.Stream(DEV), torch.cuda.Stream(DEV)
        outs_a = [torch.empty((M, Na), dtype=torch.half, device=DEV) for _ in range(24)]
        outs_b = [torch.empty((M, Nb), dtype=torch.half, device=DEV) for _ in range(24)]
        for ca, cb in zip(outs_a, outs_b):
            with torch.cuda.stream(s1):
                ext_c.gemm_half_q_half(xa, lin_a.q_handle, ca, False)
            with torch.cuda.stream(s2):
                ext_c.gemm_half_q_half(xb, lin_b.q_handle, cb, False)
        torch.cuda.synchronize()
        for ca, cb in zip(outs_a, outs_b):
            assert torch.equal(ca, want_a) and torch.equal(cb, want_b), f"M={M}: concurrent streams disturbed each other"
    lin_a.unload()
    lin_b.unload()
