#!/usr/bin/env python
"""Build the UNMODIFIED reference extension into oracle/_ref/ (test infrastructure only).

TEST INFRASTRUCTURE -- never imported by the product path (exllamav2_b200/).  Only tests/,
__graft_entry__.smoke() and bench.py's baseline legs may load what this script produces.

The reference's hot path lives in exllamav2/exllamav2_ext (C++17 + CUDA, pybind11; SURVEY.md 8c).  It
compiles from its own sources with torch's cpp_extension + ninja (no cmake, no external libs, no generated
code), so we compile the sources *where they lie* in the reference checkout with the recipe below and write the
output only into oracle/_ref/ (git-ignored build output).  No reference source is copied into this repository.
The checkout is read from /root/reference unless EXL2_REFERENCE_ROOT names another location; where neither exists
nothing is built.  The extension is compiled for sm_90a (REF_ARCH); the arch of the build in oracle/_ref/ is recorded
next to it, and a build for any other arch is replaced.  We do not run the reference's setup.py; the source list is the
directory listing of the extension (every .cpp/.cu under it), which is what setup.py:43-89 enumerates.

The module is built under the name `exllamav2_ext_ref` (the pybind module name is TORCH_EXTENSION_NAME,
ext_bindings.cpp:27), so it can be imported next to our own drop-in module.

Usage:  python oracle/build_ref.py      (about 2-3 min on 8 cores; no GPU needed)
"""
import glob
import os
import shutil
import sys

REF_ROOT = os.environ.get("EXL2_REFERENCE_ROOT") or "/root/reference"
REF_ARCH = "9.0a"                   # TORCH_CUDA_ARCH_LIST of the reference build: the H100 (sm_90a)
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
NAME = "exllamav2_ext_ref"
ARCH_STAMP = os.path.join(OUT, NAME + ".arch")


def built_arch() -> str | None:
    """The TORCH_CUDA_ARCH_LIST the extension in oracle/_ref/ was built for (None: not built, or by an unrecorded recipe)."""
    if not os.path.exists(os.path.join(OUT, NAME + ".so")) or not os.path.exists(ARCH_STAMP):
        return None
    with open(ARCH_STAMP) as f:
        return f.read().strip()


def build(verbose: bool = False) -> str | None:
    src = os.path.join(REF_ROOT, "exllamav2", "exllamav2_ext")
    target = os.path.join(OUT, NAME + ".so")
    if not os.path.isdir(src):
        return target if os.path.exists(target) else None
    if built_arch() == REF_ARCH:
        return target
    for stale in (target, ARCH_STAMP):
        if os.path.exists(stale):
            os.remove(stale)
    os.makedirs(OUT, exist_ok=True)
    os.environ["TORCH_CUDA_ARCH_LIST"] = REF_ARCH
    os.environ.setdefault("MAX_JOBS", str(os.cpu_count() or 8))
    import tempfile
    build_dir = os.path.join(tempfile.gettempdir(), f"exl2_ref_build_{REF_ARCH}")
    os.makedirs(build_dir, exist_ok=True)
    from torch.utils.cpp_extension import load

    files = sorted(
        glob.glob(os.path.join(src, "*.cpp"))
        + glob.glob(os.path.join(src, "cpp", "*.cpp"))
        + glob.glob(os.path.join(src, "cuda", "*.cu"))
        + glob.glob(os.path.join(src, "cuda", "comp_units", "*.cu"))
    )
    load(
        name=NAME,
        sources=files,
        extra_include_paths=[src],
        extra_cuda_cflags=["-lineinfo", "-O3"],
        extra_cflags=["-O3"],
        build_directory=build_dir,
        verbose=verbose,
        is_python_module=False,
    )
    shutil.copy(os.path.join(build_dir, NAME + ".so"), target)
    with open(ARCH_STAMP, "w") as f:
        f.write(REF_ARCH + "\n")
    return target


def build_pypkg() -> str | None:
    """Byte-compile the reference's PYTHON package (exllamav2/*.py: linear.py, attn.py, mlp.py, cache.py, ext.py, ... -- the
    callers of the hot path) from the sources where they lie into oracle/_ref/pypkg/exllamav2/ as sourceless .pyc files, so
    that tests/test_gpu_dropin.py can run the reference's own ExLlamaV2Linear / RMSNorm code on top of OUR extension module
    on a GPU machine without the reference checkout.  Build output only; nothing is copied into the repository."""
    import py_compile
    src = os.path.join(REF_ROOT, "exllamav2")
    dst = os.path.join(OUT, "pypkg", "exllamav2")
    stamp = os.path.join(dst, "__init__.pyc")
    if not os.path.isdir(src):
        return os.path.dirname(dst) if os.path.exists(stamp) else None
    if os.path.exists(stamp):
        return os.path.dirname(dst)
    for root, dirs, files in os.walk(src):
        dirs[:] = [d for d in dirs if d not in ("exllamav2_ext", "__pycache__")]
        rel = os.path.relpath(root, src)
        for f in files:
            if f.endswith(".py"):
                out = os.path.join(dst, rel, f + "c")
                os.makedirs(os.path.dirname(out), exist_ok=True)
                py_compile.compile(os.path.join(root, f), cfile=out, dfile=os.path.join("exllamav2", rel, f), doraise=True)
    return os.path.dirname(dst)


def load_ref():
    """Import the built reference extension (or return None when it has not been built)."""
    target = os.path.join(OUT, NAME + ".so")
    if not os.path.exists(target):
        return None
    import importlib.util

    import torch  # noqa: F401  (the extension links against libtorch)

    spec = importlib.util.spec_from_file_location(NAME, target)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    t = build(verbose="-v" in sys.argv)
    print("reference extension:", t)
    print("reference python package (byte-compiled):", build_pypkg())
