"""Build ``libxclim_b200.so`` in-tree with nvcc for sm_90a (H100; no torch, no cmake).

``python -m xclim_b200._build`` (or ``__graft_entry__.build()``) compiles every ``csrc/*.cu`` to an
object under ``build/`` and links ``xclim_b200/lib/libxclim_b200.so``.  nvcc cross-compiles without
a GPU; the built ``.so`` is git-ignored but travels to the GPU box with the repo snapshot.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB_DIR = os.path.join(PKG, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libxclim_b200.so")
OBJ_DIR = os.path.join(ROOT, "build", "obj")

#: the one target architecture: Hopper (H100, sm_90a)
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]

NVCC_FLAGS = [
    "-O3", "-std=c++17", *ARCH_FLAGS, "-lineinfo",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "--extended-lambda",
    "-Xptxas", "-v", "-Wno-deprecated-gpu-targets",
]


#: per-file flags.  fwi.cu mirrors numba / numpy arithmetic, which never fuses a multiply with an add; so does
#: dqm.cu (the trend, detrend and retrend of the oracle, operation by operation) and stdindex.cu (numpy's float32
#: moment expressions of the distribution fit) and ensemble.cu (the float64 moments and t-tests that the CPU tests
#: build for the host) and evfit.cu (numpy's float32 normal fit and the likelihood fits the CPU tests build for
#: the host) and analog.cu (the dissimilarity metrics the CPU tests build for the host) and pet.cu (the
#: evapotranspiration formulas the CPU tests build for the host).
EXTRA_FLAGS = {"fwi.cu": ["-fmad=false"], "dqm.cu": ["-fmad=false"], "stdindex.cu": ["-fmad=false"],
               "ensemble.cu": ["-fmad=false"], "evfit.cu": ["-fmad=false"], "analog.cu": ["-fmad=false"],
               "pet.cu": ["-fmad=false"], "chill.cu": ["-fmad=false"]}


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC or add /usr/local/cuda/bin to PATH)")


def sources() -> list[str]:
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def headers(*dirs: str) -> list[str]:
    """Every header under csrc/ and include/ (and under ``dirs``): what any source may include."""
    return sorted(os.path.join(d, f) for d in (CSRC, os.path.join(ROOT, "include"), *dirs)
                  for f in os.listdir(d) if f.endswith((".cuh", ".h")))


def _deps_mtime() -> float:
    # this file too: a change of NVCC_FLAGS or EXTRA_FLAGS recompiles every object
    return max(os.path.getmtime(h) for h in headers() + [os.path.abspath(__file__)])


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ_DIR, exist_ok=True)
    os.makedirs(LIB_DIR, exist_ok=True)
    hdr_m = _deps_mtime()
    # a library newer than every source and header is current even when the objects did not travel
    if not force and os.path.exists(LIB_PATH) and \
            os.path.getmtime(LIB_PATH) >= max([hdr_m] + [os.path.getmtime(s) for s in sources()]):
        return LIB_PATH
    nvcc = _nvcc()
    jobs = []
    objs = []
    for src in sources():
        obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        stale = force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hdr_m)
        if stale:
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        cmd = [nvcc, *NVCC_FLAGS, *EXTRA_FLAGS.get(os.path.basename(src), []), "-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ".ptxas.log")
        with open(log, "w") as f:
            f.write(r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(f"[build] {os.path.basename(src)} ok", file=sys.stderr)
        return obj

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(compile_one, jobs))
    need_link = force or bool(jobs) or not os.path.exists(LIB_PATH) or any(
        os.path.getmtime(o) > os.path.getmtime(LIB_PATH) for o in objs)
    if need_link:
        cmd = [nvcc, "-shared", *ARCH_FLAGS, "-o", LIB_PATH, *objs]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
