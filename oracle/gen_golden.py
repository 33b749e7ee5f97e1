#!/usr/bin/env python
"""Generate golden vectors by running the UNMODIFIED reference CUDA extension (oracle/_ref, built by
oracle/build_ref.py) on a GPU over the seeded cases of tests/cases.py.  TEST INFRASTRUCTURE.

    python oracle/gen_golden.py [outdir]        (default golden_out/; copy the .npz files to tests/golden/)

The reference has no golden vectors of its own for this path (SURVEY.md 8c); these files are what pins the CPU
oracle (tests/test_oracle_golden.py) and, on the GPU, our kernels (tests/test_gpu_golden.py,
tests/test_gpu_vs_reference.py, tests/test_gpu_row_blocks.py).
Outputs per case:  reconstruct (fp16 bits), gemm force_cuda for several M (fp16 bits; NOT bit-reproducible across
runs because the reference accumulates with fp16 atomics), plus rms_norm / rope / Q4-kv vectors, the inputs and outputs
of tests/test_gpu_vs_reference.py (ref_gemm_m4.npz: its 4-row GEMMs; ref_ops.npz: its op checks) and the 4096 x 4096 GPTQ
row of tests/test_gpu_row_blocks.py (ref_gptq_4096.npz).  ref_ops.npz stays small: the inputs are regenerated from their
seed and bit-exact outputs are stored as SHA-256 digests; the RMSNorm output (compared within 1 ulp) is stored whole.
"""
import hashlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import cases  # noqa: E402
import exl2_oracle as oracle  # noqa: E402
from build_ref import load_ref  # noqa: E402

DEV = "cuda:0"
none_tensor = torch.empty((1, 1), device="meta")


def ref_make_q_matrix(ref, w_np, prescale=1.0, offset_qzeros=False):
    """The reference's Python glue (exllamav2/ext.py:325-410, module.py:118-121) driving the reference extension."""
    w = {k: (torch.from_numpy(np.ascontiguousarray(v)) if k == "g_idx" else torch.from_numpy(np.ascontiguousarray(v)).to(DEV))
         for k, v in w_np.items()}
    if "q_weight" in w:
        w["q_perm"] = torch.argsort(w["q_invperm"]).to(torch.int)
        w["q_scale_max"] *= prescale / 256
        w["q_perm"] = w["q_perm"].short()
        w["q_invperm"] = w["q_invperm"].short()
        gm = ref.make_group_map(w["q_groups"].cpu(), w["q_weight"].shape[0]).to(DEV)
        w["q_group_map"] = gm
        K, N = w["q_perm"].shape[0], w["q_weight"].shape[1]
        temp_dq = torch.empty((K * N,), dtype=torch.half, device=DEV)
        h = ref.make_q_matrix(w["q_weight"], w["q_perm"], w["q_invperm"], w["q_scale"], w["q_scale_max"], w["q_groups"],
                              w["q_group_map"], none_tensor, none_tensor, none_tensor, w.get("bias", none_tensor), temp_dq, K)
    else:
        if offset_qzeros:
            w["qzeros"] -= 0b00010001000100010001000100010001
        K, N = w["qweight"].shape[0] * 8, w["qweight"].shape[1]
        temp_dq = torch.empty((K * N,), dtype=torch.half, device=DEV)
        if not (w["g_idx"] == 0).all().item():
            w["q_perm"] = torch.empty((K,), dtype=torch.short, device=DEV)
            w["q_invperm"] = torch.empty_like(w["q_perm"])
            h = ref.make_q_matrix(w["qweight"], w["q_perm"], w["q_invperm"], none_tensor, none_tensor, none_tensor, none_tensor,
                                  w["qzeros"], w["scales"], w["g_idx"].cpu(), w.get("bias", none_tensor), temp_dq, K)
        else:
            h = ref.make_q_matrix(w["qweight"], none_tensor, none_tensor, none_tensor, none_tensor, none_tensor, none_tensor,
                                  w["qzeros"], w["scales"], none_tensor, w.get("bias", none_tensor), temp_dq, K)
    torch.cuda.synchronize()
    return h, w, temp_dq, (K, N)


def ref_ops_inputs():
    """The seeded inputs of tests/test_gpu_vs_reference.py::test_ops_match_reference."""
    rng = np.random.default_rng(123)
    x = rng.normal(0, 1.5, size=(5, 4096)).astype(np.float16)
    w = (1 + 0.1 * rng.normal(size=(4096,))).astype(np.float16)
    rope = [rng.normal(0, 1, size=(2, 6, 8 * 128)).astype(np.float16) for _ in range(2)]    # neox, gptj
    k = rng.normal(0, 1, size=(2, 9, 8, 128)).astype(np.float16)
    v = rng.normal(0, 3, size=(2, 9, 8, 128)).astype(np.float16)
    return dict(norm_x=x, norm_w=w, rope_neox_x=rope[0], rope_gptj_x=rope[1], kv_k=k, kv_v=v)


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


def ref_ops(ref, outdir):
    """The reference's rms_norm / rope_ / Q4-kv on the seeded inputs of tests/test_gpu_vs_reference.py::test_ops_match_reference."""
    inp = ref_ops_inputs()
    out = {}
    x, w = inp["norm_x"], inp["norm_w"]
    y = torch.empty((5, 4096), dtype=torch.half, device=DEV)
    ref.rms_norm(torch.from_numpy(x).to(DEV), torch.from_numpy(w).to(DEV), y, 1e-5)
    out["norm_y"] = y.cpu().numpy().view(np.uint16)
    hd, heads = 128, 8
    sin, cos = oracle.rope_tables(hd, 128)
    st, ct = torch.from_numpy(sin).to(DEV), torch.from_numpy(cos).to(DEV)
    offs = torch.tensor([0, 11], dtype=torch.int, device=DEV)
    for neox in (True, False):
        tag = "neox" if neox else "gptj"
        xt = torch.from_numpy(inp[f"rope_{tag}_x"]).to(DEV)
        ref.rope_(xt, st, ct, 17, heads, hd, offs, neox)
        out[f"rope_{tag}_y"] = digest(xt.cpu().numpy())
    k, v = inp["kv_k"], inp["kv_v"]
    kq = torch.zeros((2, 9, 8, 64), dtype=torch.uint8, device=DEV)
    ks = torch.zeros((2, 9, 8, 4), dtype=torch.half, device=DEV)
    vq, vs = torch.zeros_like(kq), torch.zeros_like(ks)
    kt, vt = torch.from_numpy(k).to(DEV), torch.from_numpy(v).to(DEV)
    ref.fp16_to_q_kv(kt, kq, ks, vt, vq, vs, 2, 2, 6, 0, none_tensor, none_tensor, 4)
    ko, vo = torch.zeros_like(kt), torch.zeros_like(vt)
    ref.q_to_fp16_kv(kq, ko, ks, vq, vo, vs, 2, 2, 6, 0, none_tensor, none_tensor, 4)
    for name, t in (("kv_kq", kq), ("kv_ks", ks), ("kv_vq", vq), ("kv_vs", vs), ("kv_ko", ko), ("kv_vo", vo)):
        out[name] = digest(t.cpu().numpy())
    np.savez_compressed(os.path.join(outdir, "ref_ops.npz"), **out)
    print("golden ref_ops", {k: v.shape for k, v in out.items()})


def ref_gptq_4096(ref, outdir):
    """The reference's one-row GEMM on the 4096 x 4096 GPTQ g128 matrices of tests/test_gpu_row_blocks.py::test_gptq_4096_row."""
    import synth
    out = {}
    for act_order in (False, True):
        w = synth.make_gptq(4096, 4096, 128, seed=0, act_order=act_order)
        a = np.random.default_rng(0).normal(0, 1, size=(1, 4096)).astype(np.float16)
        h, keep, temp_dq, _ = ref_make_q_matrix(ref, w)
        c = torch.empty((1, 4096), dtype=torch.half, device=DEV)
        ref.gemm_half_q_half(torch.from_numpy(a).to(DEV), h, c, True)
        torch.cuda.synchronize()
        out[f"act{int(act_order)}"] = c.cpu().numpy().view(np.uint16)
        ref.free_q_matrix(h)
    np.savez_compressed(os.path.join(outdir, "ref_gptq_4096.npz"), **out)
    print("golden ref_gptq_4096", {k: v.shape for k, v in out.items()})


def main(outdir):
    ref = load_ref()
    if ref is None:
        print("oracle/_ref/exllamav2_ext_ref.so not built; run oracle/build_ref.py with EXL2_REFERENCE_ROOT set")
        return 1
    os.makedirs(outdir, exist_ok=True)
    names = [n for n in list(cases.EXL2_CASES) + list(cases.GPTQ_CASES)]
    skipped = []
    gemm_m4 = {}
    for name in names:
        K, N = cases.case_shape(name)
        if N % 32 != 0:   # the reference kernels assume 4-column vectors / 32-column tiles for these widths
            pass
        w_np = cases.make_case(name)
        try:
            h, w, temp_dq, _ = ref_make_q_matrix(ref, w_np)
        except Exception as e:  # pragma: no cover
            skipped.append((name, repr(e)))
            continue
        out = {}
        W = torch.empty((K, N), dtype=torch.half, device=DEV)
        ref.reconstruct(h, W)
        out["reconstruct"] = W.cpu().numpy().view(np.uint16)
        for M in cases.M_VALUES:
            a = torch.from_numpy(cases.activations(name, M)).to(DEV)
            c = torch.empty((M, N), dtype=torch.half, device=DEV)
            ref.gemm_half_q_half(a, h, c, True)
            out[f"gemm_m{M}"] = c.cpu().numpy().view(np.uint16)
        if N % 32 == 0:   # the 4-row GEMM of tests/test_gpu_vs_reference.py (its other row counts are in linear_<case>.npz)
            a = torch.from_numpy(cases.activations(name, 4)).to(DEV)
            c = torch.empty((4, N), dtype=torch.half, device=DEV)
            ref.gemm_half_q_half(a, h, c, True)
            gemm_m4[name] = c.cpu().numpy().view(np.uint16)
        torch.cuda.synchronize()
        ref.free_q_matrix(h)
        np.savez_compressed(os.path.join(outdir, f"linear_{name}.npz"), **out)
        print("golden", name, {k: v.shape for k, v in out.items()})

    # rms_norm / rope / kv
    rng = np.random.default_rng(77)
    ops = {}
    x = rng.normal(0, 1.5, size=(3, 2048)).astype(np.float16)
    w = (1 + 0.1 * rng.normal(size=(2048,))).astype(np.float16)
    y = torch.empty((3, 2048), dtype=torch.half, device=DEV)
    ref.rms_norm(torch.from_numpy(x).to(DEV), torch.from_numpy(w).to(DEV), y, 1e-5)
    ops["norm_x"], ops["norm_w"], ops["norm_y"] = x.view(np.uint16), w.view(np.uint16), y.cpu().numpy().view(np.uint16)
    hd, heads = 128, 4
    sin, cos = oracle.rope_tables(hd, 64)
    for neox in (True, False):
        xr = rng.normal(0, 1, size=(2, 3, heads * hd)).astype(np.float16)
        xt = torch.from_numpy(xr).to(DEV)
        offs = torch.tensor([0, 5], dtype=torch.int, device=DEV)
        ref.rope_(xt, torch.from_numpy(sin).to(DEV)[None, None], torch.from_numpy(cos).to(DEV)[None, None], 9, heads, hd, offs, neox)
        tag = "neox" if neox else "gptj"
        ops[f"rope_{tag}_x"], ops[f"rope_{tag}_y"] = xr.view(np.uint16), xt.cpu().numpy().view(np.uint16)
    ops["rope_sin"], ops["rope_cos"] = sin.view(np.uint16), cos.view(np.uint16)
    kv = rng.normal(0, 1, size=(2, 4, 8, 128)).astype(np.float16)
    kt = torch.from_numpy(kv).to(DEV)
    kq = torch.zeros((2, 4, 8, 64), dtype=torch.uint8, device=DEV)
    ks = torch.zeros((2, 4, 8, 4), dtype=torch.half, device=DEV)
    vq, vs = torch.zeros_like(kq), torch.zeros_like(ks)
    ref.fp16_to_q_kv(kt, kq, ks, kt, vq, vs, 2, 0, 4, 0, none_tensor, none_tensor, 4)
    ko, vo = torch.zeros_like(kt), torch.zeros_like(kt)
    ref.q_to_fp16_kv(kq, ko, ks, vq, vo, vs, 2, 0, 4, 0, none_tensor, none_tensor, 4)
    ops["kv_x"], ops["kv_q"], ops["kv_s"], ops["kv_y"] = kv.view(np.uint16), kq.cpu().numpy(), ks.cpu().numpy().view(np.uint16), ko.cpu().numpy().view(np.uint16)
    np.savez_compressed(os.path.join(outdir, "ops.npz"), **ops)
    print("golden ops", {k: v.shape for k, v in ops.items()})
    np.savez_compressed(os.path.join(outdir, "ref_gemm_m4.npz"), **gemm_m4)
    ref_ops(ref, outdir)
    ref_gptq_4096(ref, outdir)
    if skipped:
        print("SKIPPED:", skipped)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "golden_out")))
