"""Build libexl2b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m exllamav2_b200.build [--force] [--verbose]

The library has no torch / Python dependency (plain C ABI, include/exl2_b200.h); it is loaded with ctypes by
exllamav2_b200/ext.py.  The .so is a build product and stays out of git.
"""
from __future__ import annotations

import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libexl2b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def sources() -> list[str]:
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.h")) + glob.glob(os.path.join(CSRC, "*.cuh")) + [
        os.path.join(HERE, "..", "include", "exl2_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in sources():
        obj = os.path.join(HERE, "build", os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        extra = os.environ.get("EXL2B_NVCC_EXTRA", "").split()        # extra nvcc flags, e.g. -DNDEBUG
        cmd = [_nvcc(), *NVCC_FLAGS, *extra, "-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        log.append(f"==== {os.path.basename(src)}\n{out}")
        failed |= p.returncode != 0
    with open(os.path.join(HERE, "build", "ptxas.log"), "w") as f:
        f.write("\n".join(log))
    if failed:
        sys.stderr.write("\n".join(log))
        raise RuntimeError("nvcc failed; see exllamav2_b200/build/ptxas.log")
    if verbose:
        print("\n".join(log))
    link = [_nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB, *objs]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
