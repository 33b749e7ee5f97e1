"""The two-offset 4-bit unpack of gemm_tc_kernel (csrc/gemm_tc.cu, tc_dequant4): the tensor core multiplies the activations
with offset + q (1024 + q on even pair slots, 64 + q on odd ones) and the offsets and the zero point are removed afterwards
with two column-independent sums,   sum_k a_k (q_k - z) = D - (S1 + z * S0),   S1 = sum a_k * offset_k,  S0 = sum a_k.
Checked here in numpy with a model of the tensor core's arithmetic (exact fp16 x fp16 products, an fp32 accumulator rounded
once per k16 step): the identity holds, and with round-to-nearest the cancellation costs ~1e-5 rel-L2 for zero-mean and
shifted rows alike, far below the fp16 rounding of the output (2.8e-4 rel-L2).  The model cannot say how wgmma rounds and
aligns its accumulation: an accumulator rounding toward zero would cost ~2e-4 on shifted rows.  The GPU measurement on such
rows is tests/test_gpu_tc_paths.py::test_activation_families: on an H100, EXL2 4-bit with shifted rows gives 3.2e-4 .. 3.9e-4
rel-L2 where the dense path gives 2.1e-4 -- more than the round-to-nearest model accounts for."""
import numpy as np
import pytest


def _offsets(n_k):
    pair = (np.arange(n_k) // 2) % 16            # pair slot inside a 32-row slab
    return np.where(pair % 2 == 0, 1024.0, 64.0).astype(np.float32)


@pytest.mark.parametrize("z", [8, 1, 16])        # EXL2 zero point 8; GPTQ z + 1 in 1..16
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_two_offset_identity(z, seed):
    rng = np.random.default_rng(seed)
    K, N = 128, 64                               # one quantisation group, 64 weight columns
    a = rng.normal(0, 1, size=(K,)).astype(np.float16)
    q = rng.integers(0, 16, size=(K, N))
    off = _offsets(K)
    A = (off[:, None] + q).astype(np.float16)    # what the unpack stores: exactly representable (<= 1039)
    assert np.array_equal(A.astype(np.float32), off[:, None] + q)
    prod = a.astype(np.float32)[:, None] * A.astype(np.float32)          # exact in fp32 (11 x 11 significant bits)
    D = np.zeros((N,), dtype=np.float32)
    for k in range(K):                           # fp32 accumulation, in order
        D += prod[k]
    a32 = a.astype(np.float32)
    S1 = np.float32(0)
    S0 = np.float32(0)
    for k in range(K):
        S1 = np.float32(S1 + a32[k] * off[k])
        S0 = np.float32(S0 + a32[k])
    got = D - (S1 + np.float32(z) * S0)
    want = (a.astype(np.float64)[:, None] * (q - z)).sum(0)
    scale = np.abs(a.astype(np.float64)).sum() * 8.0                    # what sum |a| |q - z| can reach
    assert np.max(np.abs(got - want)) < 2e-5 * scale * 128              # fp32 epsilon times the 1024-offset partial sums
    assert np.max(np.abs(got - want)) < 0.05 * np.std(want)             # and negligible against the result itself


def _round_f32(x, toward_zero):
    r = x.astype(np.float32)
    if toward_zero:
        r = np.where(np.abs(r.astype(np.float64)) > np.abs(x), np.nextafter(r, np.float32(0)), r).astype(np.float32)
    return r


def _model_rel_l2(mu, toward_zero, G=32, N=256, seed=0):
    """A K = 128 G row of mean mu through the two-offset form, with the accumulator rounded to fp32 once per k16 step (exact
    products, exact sum within the step) either to nearest or toward zero; per-group scales applied in fp32.  Returns the
    rel-L2 of the result vs fp64."""
    rng = np.random.default_rng(seed)
    K = 128 * G
    a = rng.normal(mu, 1, size=K).astype(np.float16).astype(np.float64)
    q = rng.integers(0, 16, size=(K, N))
    off = _offsets(K).astype(np.float64)
    scale = rng.uniform(0.5, 1.5, size=(G, N)).astype(np.float32)
    tot = np.zeros(N, np.float32)
    for g in range(G):
        sl = slice(128 * g, 128 * g + 128)
        A = off[sl, None] + q[sl]
        D = np.zeros(N, np.float32)
        for k0 in range(0, 128, 16):
            D = _round_f32(D.astype(np.float64) + (a[sl][k0:k0 + 16, None] * A[k0:k0 + 16]).sum(0), toward_zero)
        S1 = np.float32((a[sl] * off[sl]).sum())
        S0 = np.float32(a[sl].sum())
        tot = np.float32(tot + scale[g] * (D - (S1 + np.float32(8) * S0)))
    want = sum(scale[g].astype(np.float64) * (a[128 * g:128 * g + 128, None] * (q[128 * g:128 * g + 128] - 8)).sum(0) for g in range(G))
    return float(np.linalg.norm(tot - want) / np.linalg.norm(want))


@pytest.mark.parametrize("mu", [0.0, 1.0, 2.0, 4.0])
def test_two_offset_shifted_rows_model(mu):
    """Rows with a DC component (mu != 0) leave a large D = sum a (offset + q) that the per-group correction cancels.  With a
    round-to-nearest fp32 accumulator the cancellation costs ~1e-5 rel-L2 at every mean; an accumulator that rounds toward zero
    (or truncates alignment bits) would bias every step the same way: ~2e-4 for mu >= 1, 40 % of the 5e-4 contract.
    tests/test_gpu_tc_paths.py::test_activation_families measures what the tensor core does on such rows."""
    rn, rz = _model_rel_l2(mu, False), _model_rel_l2(mu, True)
    assert rn < 3e-5, f"round to nearest: {rn:.2e}"
    assert rz < 4e-4, f"round toward zero: {rz:.2e}"
    if mu >= 1:
        assert rz > 5 * rn, f"toward zero {rz:.2e} vs nearest {rn:.2e}: the model no longer separates the two"
