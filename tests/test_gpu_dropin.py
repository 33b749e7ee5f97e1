"""The drop-in, EXECUTED: the reference's own Python modules (exllamav2/linear.py, rmsnorm.py, ext.py -- byte-compiled from
the reference checkout into oracle/_ref/pypkg by oracle/build_ref.py, so that the GPU machine needs no checkout) run
on top of exllamav2_b200.ext installed under the name the reference imports (`exllamav2_ext`, exllamav2/ext.py:106-109).

  * ExLlamaV2Linear.load(dict) -> ext.make_q_matrix (ext.py:325-410) -> our make_q_matrix, EXL2 and GPTQ (+ act-order);
    forward() -> ext_c.gemm_half_q_half (linear.py:366); get_weight_tensor_dq() -> ext_c.reconstruct (linear.py:493);
    results vs the numpy oracle (reconstruct bit-exact, forward <= 1e-3 for 1 .. 40 rows);
  * ExLlamaV2RMSNorm.forward -> ext_c.rms_norm (rmsnorm.py:141);
  * names outside the hot path reach the registered stock extension through the module-level forwarder, or raise an
    AttributeError that says so.
The first two skip when oracle/_ref/pypkg has not been built (python oracle/build_ref.py); the forwarder test registers a
stand-in stock module when the reference extension is not built.
"""
import os
import sys
import types

import numpy as np
import pytest
import torch

import cases
import exl2_oracle as oracle

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PYPKG = os.path.join(ROOT, "oracle", "_ref", "pypkg")


@pytest.fixture(scope="module")
def ref_py():
    if not os.path.exists(os.path.join(PYPKG, "exllamav2", "__init__.pyc")):
        pytest.skip("oracle/_ref/pypkg not built (python oracle/build_ref.py)")
    import exllamav2_b200.ext as b200_ext
    b200_ext.install_as_exllamav2_ext()              # INTEGRATION.md section 1: before `import exllamav2`
    sys.path.insert(0, PYPKG)
    import exllamav2                                  # noqa: F401  the reference package, unmodified
    from exllamav2 import ext as ref_ext
    assert ref_ext.ext_c is b200_ext, "the reference did not pick up the drop-in module"
    return types.SimpleNamespace(ext=ref_ext, b200=b200_ext)


def _stub_model():
    """What ExLlamaV2Linear / ExLlamaV2RMSNorm read from their model: a config (linear.py:128-167, rmsnorm.py:56-60)."""
    arch = types.SimpleNamespace(norm_constant_bias=0)
    cfg = types.SimpleNamespace(load_in_q4=False, max_dq_size=512 * 1024 * 1024, checkpoint_offset_qzeros=False, norm_eps=1e-5,
                                max_input_len=2048, max_batch_size=1, arch=types.SimpleNamespace(lm=arch))
    return types.SimpleNamespace(config=cfg), arch


def _tensors(w_np):
    return {k: (torch.from_numpy(np.ascontiguousarray(v)) if k == "g_idx" else torch.from_numpy(np.ascontiguousarray(v)).to(DEV))
            for k, v in w_np.items()}


@pytest.mark.parametrize("name", ["b4_g128", "b54_g64", "b865_mixed", "b6_g128_bias", "gptq_g128", "gptq_g128_act", "gptq_g64_act_b"])
def test_reference_linear_on_dropin(ref_py, name):
    from exllamav2.linear import ExLlamaV2Linear
    w_np = cases.make_case(name)
    K, N = cases.case_shape(name)
    model, arch = _stub_model()
    lin = ExLlamaV2Linear(model, "model.layers.0.self_attn.q_proj", K, N, "bias" in w_np, archparams=arch)
    lin.device_idx = 0
    w = _tensors(w_np)
    if "q_invperm" in w:
        w["q_perm"] = torch.argsort(w["q_invperm"]).to(torch.int)      # what the loader derives, module.py:118-121
    lin.load(w, device_context=False)
    assert lin.q_handle
    W = oracle.exl2_reconstruct(w_np) if name in cases.EXL2_CASES else oracle.gptq_reconstruct(w_np)
    got_w = lin.get_weight_tensor_dq()
    assert np.array_equal(cases.u16(got_w.cpu().numpy()), cases.u16(W))
    for M in (1, 5, 40):
        a = cases.activations(name, M)
        y = lin.forward(torch.from_numpy(a).to(DEV), force_cuda=True)
        truth = oracle.gemm_truth(a, W, w_np.get("bias"))
        err = oracle.rel_l2(y.cpu().numpy(), truth)
        assert err <= 1e-3, f"{name} M={M}: {err:.2e}"
    lin.unload()
    assert lin.q_handle is None


def test_reference_rmsnorm_on_dropin(ref_py):
    from exllamav2.rmsnorm import ExLlamaV2RMSNorm
    model, arch = _stub_model()
    norm = ExLlamaV2RMSNorm(model, "model.norm", archparams=arch)
    rng = np.random.default_rng(3)
    w = (1 + 0.1 * rng.normal(size=(4096,))).astype(np.float16)
    x = rng.normal(0, 1.5, size=(3, 4096)).astype(np.float16)
    norm.weight = torch.nn.Parameter(torch.from_numpy(w).to(DEV), requires_grad=False)
    norm.variance_epsilon = 1e-5
    y = norm.forward(torch.from_numpy(x).to(DEV))
    want = oracle.rms_norm(x, w, 1e-5)

    def key(t):
        u = np.ascontiguousarray(t, dtype=np.float16).view(np.uint16).astype(np.int32)
        return np.where(u & 0x8000, -(u & 0x7FFF), u & 0x7FFF)
    assert np.abs(key(y.cpu().numpy()) - key(want)).max() <= 1


def _stand_in_stock():
    """A module exporting two of the stock extension's out-of-scope names with its semantics: tensor_remap permutes the
    columns of a 2-D int32 tensor in place (ext_stloader.cpp:159-219), sample_basic is only looked up."""
    m = types.ModuleType("exllamav2_ext_stock")

    def tensor_remap(t, idx):
        t.copy_(t[:, idx.long()])

    def sample_basic(*args):
        raise NotImplementedError

    m.tensor_remap, m.sample_basic = tensor_remap, sample_basic
    return m


def test_out_of_scope_names_forward_to_stock():
    """Names outside the hot path reach the registered stock extension through the module-level forwarder (the reference's
    own build when oracle/_ref has it, else a stand-in module), or raise an AttributeError that says so."""
    import exllamav2_b200.ext as b
    b.install_as_exllamav2_ext()
    import exllamav2_ext                               # the name the reference's exllamav2/ext.py imports
    assert exllamav2_ext is b
    b.set_stock_extension(None)
    with pytest.raises(AttributeError, match="outside the quantized-linear hot path"):
        b.sample_basic
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    from build_ref import load_ref
    stock = load_ref() or _stand_in_stock()
    b.set_stock_extension(stock)
    try:
        assert b.sample_basic is stock.sample_basic            # exllamav2/generator/sampler.py calls ext_c.sample_basic
        # an out-of-scope op actually runs through the forwarder: tensor_remap (ext_stloader.cpp:159-219, linear.py:157)
        t = torch.arange(8 * 4, dtype=torch.int32).view(8, 4).contiguous()
        idx = torch.tensor([3, 2, 1, 0], dtype=torch.int32)
        want = t[:, idx.long()].clone()
        exllamav2_ext.tensor_remap(t, idx)
        assert torch.equal(t, want)
    finally:
        b.set_stock_extension(None)
