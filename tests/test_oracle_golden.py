"""Pin the CPU oracle against golden vectors produced by the UNMODIFIED reference CUDA extension
(oracle/gen_golden.py -> tests/golden/*.npz).  Runs without a GPU."""
import glob
import os

import numpy as np
import pytest

import cases
import exl2_oracle as oracle

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LINEAR = sorted(os.path.basename(p)[len("linear_"):-4] for p in glob.glob(os.path.join(GOLD, "linear_*.npz")))


def _ulp(a, b):
    def key(x):
        u = np.ascontiguousarray(x).view(np.uint16).astype(np.int32)
        return np.where(u & 0x8000, -(u & 0x7FFF), u & 0x7FFF)
    return np.abs(key(a) - key(b))


def test_golden_files_present():
    assert len(LINEAR) >= 12 and os.path.exists(os.path.join(GOLD, "ops.npz"))


@pytest.mark.parametrize("name", LINEAR)
def test_reconstruct_bit_exact_vs_reference(name):
    g = np.load(os.path.join(GOLD, f"linear_{name}.npz"))
    w = cases.make_case(name)
    W = oracle.exl2_reconstruct(w) if name in cases.EXL2_CASES else oracle.gptq_reconstruct(w)
    assert np.array_equal(W.view(np.uint16), g["reconstruct"]), f"{name}: oracle reconstruct differs from the reference"


@pytest.mark.parametrize("name", LINEAR)
def test_gemm_truth_vs_reference_kernel(name):
    """The reference GEMV accumulates in fp16 with atomics (q_gemm_kernel.cuh:95-113,560), so it is only ~1e-3
    accurate; the oracle's fp64 truth must sit within that of the reference's own output."""
    g = np.load(os.path.join(GOLD, f"linear_{name}.npz"))
    w = cases.make_case(name)
    W = oracle.exl2_reconstruct(w) if name in cases.EXL2_CASES else oracle.gptq_reconstruct(w)
    for M in cases.M_VALUES:
        truth = oracle.gemm_truth(cases.activations(name, M), W, w.get("bias"))
        ref = g[f"gemm_m{M}"].view(np.float16)
        assert oracle.rel_l2(ref, truth) <= 3e-3, f"{name} M={M}"


def test_ops_vs_reference():
    g = np.load(os.path.join(GOLD, "ops.npz"))
    f16 = lambda k: g[k].view(np.float16)
    # rms_norm: <= 1 ulp (fp32 summation order)
    y = oracle.rms_norm(f16("norm_x"), f16("norm_w"), 1e-5)
    assert _ulp(y, f16("norm_y")).max() <= 1
    # rope: bit-exact
    sin, cos = f16("rope_sin"), f16("rope_cos")
    s2, c2 = oracle.rope_tables(128, 64)
    assert np.array_equal(s2.view(np.uint16), g["rope_sin"]) and np.array_equal(c2.view(np.uint16), g["rope_cos"])
    for tag, fn in (("neox", oracle.rope_neox), ("gptj", oracle.rope_gptj)):
        x = f16(f"rope_{tag}_x")
        offs = [0, 5]
        want = np.stack([fn(x[b].reshape(3, 4, 128), sin, cos, 9 + offs[b] + np.arange(3)).reshape(3, 512) for b in range(2)])
        assert np.array_equal(want.view(np.uint16), g[f"rope_{tag}_y"]), tag
    # Q4 kv: scales exact; nibbles equal except rounding ties of the rcp-based division; unpack exact given q
    x = f16("kv_x").reshape(2, -1)
    pq, ps = oracle.kv_pack_q4(x)
    assert np.array_equal(ps.view(np.uint16).reshape(-1), g["kv_s"].reshape(-1))
    gq = g["kv_q"].reshape(2, -1)
    d_lo = (pq & 15).astype(int) - (gq & 15).astype(int)
    d_hi = (pq >> 4).astype(int) - (gq >> 4).astype(int)
    assert np.abs(d_lo).max() <= 1 and np.abs(d_hi).max() <= 1
    assert np.count_nonzero(d_lo) + np.count_nonzero(d_hi) <= 1e-3 * x.size
    y = oracle.kv_unpack_q4(gq, g["kv_s"].view(np.float16).reshape(2, -1))
    assert np.array_equal(y.view(np.uint16).reshape(-1), g["kv_y"].reshape(-1))
