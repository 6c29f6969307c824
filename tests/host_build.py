"""TEST INFRASTRUCTURE: compile a host build of the device code (a shim under tests/csrc/) and bind it.

The library goes to ``<tmp>/xclim_b200_host/<name>-<key>.so``, where the key hashes the compiler command, the shim
and every header of the tree: editing any header rebuilds, and two checkouts never load each other's builds."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

from xclim_b200 import _build

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc")
CUDA_INCLUDE = "/usr/local/cuda/include"
_handles = {}


def _command(src, nvcc, flags):
    if nvcc:
        cmd = [_build._nvcc(), "-O2", "-std=c++17", *_build.ARCH_FLAGS, "-Xcompiler", "-fPIC", "-shared"]
    else:
        cmd = ["g++", *(["-I" + CUDA_INCLUDE] if os.path.isdir(CUDA_INCLUDE) else []),
               "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared"]
    return cmd + list(flags) + [src]


def load(name, source, *, nvcc=False, flags=(), signatures=None):
    """The host build of ``tests/csrc/<source>`` (g++, or nvcc with ``nvcc=True``; ``flags`` appended), with
    ``signatures`` (symbol -> (restype, argtypes)) applied.  Compiles only when no build of this key exists."""
    src = os.path.join(CSRC, source)
    cmd = _command(src, nvcc, flags)
    h = hashlib.sha256("\0".join(cmd).encode())
    for path in [src] + _build.headers(CSRC):
        with open(path, "rb") as f:
            h.update(path.encode() + b"\0" + f.read())
    key = h.hexdigest()[:16]
    if (name, key) not in _handles:
        out = os.path.join(tempfile.gettempdir(), "xclim_b200_host", f"{name}-{key}.so")
        if not os.path.exists(out):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            tmp = f"{out}.{os.getpid()}.tmp"
            r = subprocess.run(cmd + ["-o", tmp], capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"host build of {source} failed:\n{' '.join(cmd)}\n{r.stdout}{r.stderr}")
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        for sym, (res, args) in (signatures or {}).items():
            fn = getattr(lib, sym)
            fn.restype, fn.argtypes = res, args
        _handles[name, key] = lib
    return _handles[name, key]
