"""GPU cross-check against the UNMODIFIED reference extension on identical tensors -- SURVEY.md 8c row (iv).  What the
reference computed is stored under tests/golden/ by oracle/gen_golden.py (seeded cases of tests/cases.py):
linear_<case>.npz (reconstruct, gemm_m<M>), ref_gemm_m4.npz (4-row GEMMs), ref_ops.npz (rms_norm / rope / Q4 kv of the
seeded inputs of oracle/gen_golden.py:ref_ops_inputs; bit-exact outputs as SHA-256 digests).

Contract (SURVEY.md 8c tolerance row):
  reconstruct                bit-exact
  gemm (M <= 32, force_cuda) rel_l2(new, ref) <= 1e-3  and  rel_l2(new, truth) <= rel_l2(ref, truth) + 1e-5
  rms_norm                   <= 1 fp16 ulp;   rope: bit-exact;   Q4 kv pack/unpack: bit-exact (same intrinsics)
"""
import hashlib
import os

import numpy as np
import pytest
import torch

import cases
import exl2_oracle as oracle

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _gold(name):
    return np.load(os.path.join(GOLD, name))


def _mine(name):
    from exllamav2_b200.linear import ExLlamaV2Linear, load_tensor_dict
    w_np = cases.make_case(name)
    K, N = cases.case_shape(name)
    lin = ExLlamaV2Linear(K, N, has_bias="bias" in w_np, device=DEV)
    lin.load(load_tensor_dict(w_np, DEV))
    return lin, w_np


# the reference's kernels need N % 32 == 0 style tiles; keep to the shapes it supports
REF_CASES = [n for n in list(cases.EXL2_CASES) + list(cases.GPTQ_CASES) if cases.case_shape(n)[1] % 32 == 0]


@pytest.mark.parametrize("name", REF_CASES)
def test_reconstruct_matches_reference(name):
    lin, w_np = _mine(name)
    W_ref = _gold(f"linear_{name}.npz")["reconstruct"]
    W_new = lin.get_weight_tensor_dq().cpu().numpy()
    assert np.array_equal(W_ref, cases.u16(W_new))
    lin.unload()


@pytest.mark.parametrize("name", REF_CASES)
@pytest.mark.parametrize("M", [1, 4, 8, 19])
def test_gemm_matches_reference(name, M):
    lin, w_np = _mine(name)
    a = cases.activations(name, M)
    at = torch.from_numpy(a).to(DEV)
    c_ref = (_gold("ref_gemm_m4.npz")[name] if M == 4 else _gold(f"linear_{name}.npz")[f"gemm_m{M}"]).view(np.float16)
    c_new = lin.forward(at)
    W = oracle.exl2_reconstruct(w_np) if name in cases.EXL2_CASES else oracle.gptq_reconstruct(w_np)
    truth = oracle.gemm_truth(a, W, w_np.get("bias"))
    e_ref = oracle.rel_l2(c_ref, truth)
    e_new = oracle.rel_l2(c_new.cpu().numpy(), truth)
    e_x = oracle.rel_l2(c_new.cpu().numpy(), c_ref.astype(np.float32))
    assert e_x <= 1e-3 + e_ref, f"new vs ref {e_x:.2e} (ref vs truth {e_ref:.2e})"
    assert e_new <= e_ref + 1e-5, f"new {e_new:.2e} is further from truth than ref {e_ref:.2e}"
    lin.unload()


def _digest(t):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(t.cpu().numpy()).tobytes()).digest(), dtype=np.uint8)


def test_ops_match_reference():
    from gen_golden import ref_ops_inputs

    from exllamav2_b200 import ext as ext_c
    from exllamav2_b200.ext import none_tensor
    g = _gold("ref_ops.npz")
    inp = ref_ops_inputs()
    f16 = lambda k: torch.from_numpy(inp[k]).to(DEV)
    # rms_norm
    x, w = f16("norm_x"), f16("norm_w")
    y_new = torch.empty_like(x)
    ext_c.rms_norm(x, w, y_new, 1e-5)
    y_ref = torch.from_numpy(g["norm_y"].view(np.int16)).to(DEV)
    diff = (y_ref.int() - y_new.view(torch.int16).int()).abs()
    assert diff.max().item() <= 1
    # rope (both styles), with per-batch offsets
    hd, heads = 128, 8
    sin, cos = oracle.rope_tables(hd, 128)
    st, ct = torch.from_numpy(sin).to(DEV), torch.from_numpy(cos).to(DEV)
    offs = torch.tensor([0, 11], dtype=torch.int, device=DEV)
    for neox in (True, False):
        tag = "neox" if neox else "gptj"
        b = f16(f"rope_{tag}_x")
        ext_c.rope_(b, st, ct, 17, heads, hd, offs, neox)
        assert np.array_equal(g[f"rope_{tag}_y"], _digest(b)), f"rope neox={neox}"
    # Q4 kv
    k, v = f16("kv_k"), f16("kv_v")
    kq = torch.zeros((2, 9, 8, 64), dtype=torch.uint8, device=DEV)
    ks = torch.zeros((2, 9, 8, 4), dtype=torch.half, device=DEV)
    vq, vs = torch.zeros_like(kq), torch.zeros_like(ks)
    ext_c.fp16_to_q_kv(k, kq, ks, v, vq, vs, 2, 2, 6, 0, none_tensor, none_tensor, 4)
    ko, vo = torch.zeros_like(k), torch.zeros_like(v)
    ext_c.q_to_fp16_kv(kq, ko, ks, vq, vo, vs, 2, 2, 6, 0, none_tensor, none_tensor, 4)
    for name, t in (("kv_kq", kq), ("kv_ks", ks), ("kv_vq", vq), ("kv_vs", vs), ("kv_ko", ko), ("kv_vo", vo)):
        assert np.array_equal(g[name], _digest(t)), name
