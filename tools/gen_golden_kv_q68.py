#!/usr/bin/env python
"""Write tests/golden/ref_kv_q68.npz: the Q6 / Q8 cache pack and unpack of the UNMODIFIED reference extension (oracle/_ref,
built by oracle/build_ref.py) on the seeded cases of tests/kv_q68.py.  Needs a GPU.

    python tools/gen_golden_kv_q68.py [outdir]        (default golden_out/; copy the .npz file to tests/golden/)

Per case and wbits (6, 8), keys `<case>_w<wbits>_<item>`:
  non-paged: kq ks vq vs   the packed bytes and scales of the whole tensors (zero-initialised), stored whole
             ko vo         SHA-256 of q_to_fp16_kv of those bytes over the same token range (zero-initialised output)
  paged:     kq ks vq vs   SHA-256 of the whole paged tensors after the pack
             kq_rows ...   the rows the pack converted, gathered in paged_rows() order, stored whole
             ko vo         SHA-256 of q_to_fp16_kv over [0, seqlen + q_len) of every sequence
The inputs are regenerated from their seeds, so the file stays small."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import kv_q68  # noqa: E402
from build_ref import load_ref  # noqa: E402

DEV = "cuda:0"
none_tensor = torch.empty((1, 1), device="meta")


def _zeros_like_state(x, bits):
    shp = tuple(x.shape[:-1])
    return (torch.zeros(shp + (x.shape[-1] * bits // 8,), dtype=torch.uint8, device=DEV),
            torch.zeros(shp + (x.shape[-1] // 32,), dtype=torch.half, device=DEV))


def nonpaged(ref, name, wbits, out):
    c = kv_q68.NONPAGED[name]
    kb, vb = kv_q68.widths(wbits)
    k, v = kv_q68.nonpaged_inputs(name)
    kt, vt = torch.from_numpy(k).to(DEV), torch.from_numpy(v).to(DEV)
    kq, ks = _zeros_like_state(kt, kb)
    vq, vs = _zeros_like_state(vt, vb)
    B = c["shape"][0]
    ref.fp16_to_q_kv(kt, kq, ks, vt, vq, vs, B, c["offset"], c["width"], 0, none_tensor, none_tensor, wbits)
    ko, vo = torch.zeros_like(kt), torch.zeros_like(vt)
    ref.q_to_fp16_kv(kq, ko, ks, vq, vo, vs, B, c["offset"], c["width"], 0, none_tensor, none_tensor, wbits)
    torch.cuda.synchronize()
    tag = f"{name}_w{wbits}_"
    out[tag + "kq"], out[tag + "vq"] = kq.cpu().numpy(), vq.cpu().numpy()
    out[tag + "ks"], out[tag + "vs"] = ks.cpu().numpy().view(np.uint16), vs.cpu().numpy().view(np.uint16)
    out[tag + "ko"], out[tag + "vo"] = kv_q68.digest(ko.cpu().numpy()), kv_q68.digest(vo.cpu().numpy())


def paged(ref, name, wbits, out):
    c = kv_q68.PAGED[name]
    kb, vb = kv_q68.widths(wbits)
    k, v = kv_q68.paged_inputs(name)
    kt, vt = torch.from_numpy(k).to(DEV), torch.from_numpy(v).to(DEV)
    kq, ks = _zeros_like_state(kt, kb)
    vq, vs = _zeros_like_state(vt, vb)
    bt = torch.tensor(c["block_table"], dtype=torch.int32, device=DEV)
    sl = torch.tensor(c["seqlens"], dtype=torch.int32, device=DEV)
    B = bt.shape[0]
    ref.fp16_to_q_kv(kt, kq, ks, vt, vq, vs, B, 0, c["q_len"], kv_q68.PAGE, sl, bt, wbits)
    ko, vo = torch.zeros_like(kt), torch.zeros_like(vt)
    ref.q_to_fp16_kv(kq, ko, ks, vq, vo, vs, B, 0, 0, kv_q68.PAGE, sl + c["q_len"], bt, wbits)
    torch.cuda.synchronize()
    tag = f"{name}_w{wbits}_"
    rows = kv_q68.paged_rows(name)
    pg = np.array([r[2] for r in rows])
    rr = np.array([r[3] for r in rows])
    for item, t in (("kq", kq), ("ks", ks), ("vq", vq), ("vs", vs)):
        a = t.cpu().numpy()
        a = a.view(np.uint16) if a.dtype == np.float16 else a
        out[tag + item] = kv_q68.digest(a)
        out[tag + item + "_rows"] = a[pg, rr]
    out[tag + "ko"], out[tag + "vo"] = kv_q68.digest(ko.cpu().numpy()), kv_q68.digest(vo.cpu().numpy())


def main(outdir):
    ref = load_ref()
    if ref is None:
        print("oracle/_ref/exllamav2_ext_ref.so not built; run oracle/build_ref.py with EXL2_REFERENCE_ROOT set")
        return 1
    os.makedirs(outdir, exist_ok=True)
    out = {}
    for wbits in (6, 8):
        for name in kv_q68.NONPAGED:
            nonpaged(ref, name, wbits, out)
        for name in kv_q68.PAGED:
            paged(ref, name, wbits, out)
    path = os.path.join(outdir, "ref_kv_q68.npz")
    np.savez_compressed(path, **out)
    print("golden", path, sum(a.nbytes for a in out.values()), "bytes,", len(out), "arrays")
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "golden_out")))
