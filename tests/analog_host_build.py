"""TEST INFRASTRUCTURE: build and bind the host build of the spatial-analogue device code
(tests/csrc/analog_host.cpp over xclim_b200/csrc/analog_core.cuh)."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
_lib = None
_vp, _i64, _i32, _f64 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_double

METHODS = {"seuclidean": 0, "nearest_neighbor": 1, "zech_aslan": 2, "szekely_rizzo": 3, "kolmogorov_smirnov": 4,
           "kldiv": 5, "mahalanobis": 6}
STATUS_NOT_FINITE, STATUS_CHKFINITE = 1, 2


def load():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.gettempdir(), f"libxclim_b200_analog_host_{os.getuid()}.so")
        src = os.path.join(HERE, "csrc", "analog_host.cpp")
        deps = [src, os.path.join(ROOT, "include", "xclim_b200.h"),
                os.path.join(ROOT, "xclim_b200", "csrc", "analog_core.cuh")]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
            tmp = out + f".{os.getpid()}.tmp"
            cmd = ["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", src, "-o", tmp]
            subprocess.run(cmd, check=True, capture_output=True, text=True)
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        lib.an_host_analog.restype = _i32
        lib.an_host_analog.argtypes = [_vp, _i32, _i32, _vp, _i32, _i64, _i32, _i32, _f64, _vp, _vp]
        _lib = lib
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def analog(target, cand, method, param=0.0, consts=None):
    """target (K, n, d), cand (C, m, d), consts (K, ...) float64 or None -> ((K, C) float64, status)."""
    t = np.ascontiguousarray(target, dtype=np.float64)
    y = np.ascontiguousarray(cand, dtype=np.float64)
    K, n, d = t.shape
    C, m, _ = y.shape
    cst = None if consts is None else np.ascontiguousarray(consts, dtype=np.float64)
    out = np.empty((K, C))
    st = load().an_host_analog(_p(t), n, K, _p(y), m, C, d, METHODS[method], float(param), _p(cst), _p(out))
    return out, int(st)
