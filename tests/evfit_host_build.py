"""TEST INFRASTRUCTURE: build and bind the host build of the frequency-analysis device code
(tests/csrc/evfit_host.cpp over xclim_b200/csrc/evfit_core.cuh)."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
_lib = None
_vp, _i64, _i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32

DISTS = {"norm": 0, "gumbel_r": 1, "genextreme": 2}
KINDS = {"ppf": 0, "isf": 1, "cdf": 2}


def load():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.gettempdir(), f"libxclim_b200_evfit_host_{os.getuid()}.so")
        src = os.path.join(HERE, "csrc", "evfit_host.cpp")
        csrc = os.path.join(ROOT, "xclim_b200", "csrc")
        deps = [src, os.path.join(ROOT, "include", "xclim_b200.h")] + \
            [os.path.join(csrc, f) for f in ("evfit_core.cuh", "normal_core.cuh", "npsum.cuh")]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
            tmp = out + f".{os.getpid()}.tmp"
            cmd = ["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", src, "-o", tmp]
            subprocess.run(cmd, check=True, capture_output=True, text=True)
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        lib.ev_host_fit.restype = _i32
        lib.ev_host_fit.argtypes = [_vp, _i64, _i64, _i64, _i32, _vp, _vp]
        lib.ev_host_transform.restype = None
        lib.ev_host_transform.argtypes = [_vp, _i64, _i32, _i32, _vp, _i32, _vp]
        lib.ev_host_gev_derivs.restype = None
        lib.ev_host_gev_derivs.argtypes = [_vp, _i32, _vp, _vp, _vp]
        _lib = lib
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def fit(x, dist):
    """(T, C) float32 -> ((2 | 3, C) float64 params, status) through the host build of fit_cell."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    T, C = x.shape
    params = np.empty((3 if dist == "genextreme" else 2, C))
    ws = np.empty(T * C, np.float32)
    st = load().ev_host_fit(_p(x), T, C, C, DISTS[dist], _p(params), _p(ws))
    return params, int(st)


def transform(params, dist, kind, q):
    params = np.ascontiguousarray(params, dtype=np.float64)
    q = np.ascontiguousarray(np.atleast_1d(q), dtype=np.float64)
    C = params.shape[1]
    out = np.empty((q.size, C))
    load().ev_host_transform(_p(params), C, DISTS[dist], KINDS[kind], _p(q), q.size, _p(out))
    return out


def gev_derivs(x, theta):
    x = np.ascontiguousarray(x, dtype=np.float32)
    th = np.ascontiguousarray(theta, dtype=np.float64)
    g, H = np.empty(3), np.empty(9)
    load().ev_host_gev_derivs(_p(x), x.size, _p(th), _p(g), _p(H))
    return g, H.reshape(3, 3)
