"""In-tree build of libtdb200.so (sm_90a only).  nvcc cross-compiles without a GPU.

    python -m turbodiffusion_b200._build [--force]

Objects go to turbodiffusion_b200/csrc/build/, the library to turbodiffusion_b200/libtdb200.so (both git-ignored
build products).  cudart is linked statically so the library has no load-time dependency on
a particular libcudart.so; the driver entry point for cuTensorMapEncodeTiled is resolved at run time.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import shutil
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
BUILD = os.path.join(CSRC, "build")
LIB_PATH = os.path.join(PKG_DIR, "libtdb200.so")
INCLUDE = os.path.join(os.path.dirname(PKG_DIR), "include")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
]


def _extra_defines():
    """Extra nvcc defines for experimental kernel variants (TDB200_NVCC_DEFINES="-DNAME=VALUE ..."); unset = the shipped kernels.
    Changing it needs --force (object staleness only tracks source mtimes)."""
    return os.environ.get("TDB200_NVCC_DEFINES", "").split()


def _nvcc() -> str:
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found; libtdb200.so cannot be built")
    return nvcc


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(BUILD, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(INCLUDE, "tdb200.h"))
    nvcc = _nvcc()
    jobs = []
    for src in sources():
        obj = os.path.join(BUILD, src[:-3] + ".o")
        if force or _stale(obj, [os.path.join(CSRC, src)] + headers):
            cmd = [nvcc] + NVCC_FLAGS + _extra_defines() + (["-Xptxas", "-v"] if verbose else []) + ["-I", INCLUDE, "-c",
                                                                                  os.path.join(CSRC, src), "-o", obj]
            jobs.append((src, cmd))
    if jobs:
        with cf.ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            futs = {ex.submit(subprocess.run, cmd, capture_output=True, text=True): src for src, cmd in jobs}
            for fut in cf.as_completed(futs):
                r = fut.result()
                if verbose and r.stderr:
                    print(r.stderr, file=sys.stderr)
                if r.returncode != 0:
                    raise RuntimeError(f"nvcc failed on {futs[fut]}:\n{r.stdout}\n{r.stderr}")
    objs = [os.path.join(BUILD, s[:-3] + ".o") for s in sources()]
    if force or jobs or _stale(LIB_PATH, objs):
        cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB_PATH] + objs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
