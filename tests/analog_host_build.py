"""TEST INFRASTRUCTURE: build and bind the host build of the spatial-analogue device code
(tests/csrc/analog_host.cpp over xclim_b200/csrc/analog_core.cuh)."""
import ctypes

import numpy as np

import host_build
from xclim_b200 import _lib as L

_vp, _i64, _i32, _f64 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_double
SIGNATURES = {"an_host_analog": (_i32, [_vp, _i32, _i32, _vp, _i32, _i64, _i32, _i32, _f64, _vp, _vp])}


def load():
    return host_build.load("analog", "analog_host.cpp", signatures=SIGNATURES)


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
    st = load().an_host_analog(_p(t), n, K, _p(y), m, C, d, L.AN_METHODS[method], float(param), _p(cst), _p(out))
    return out, int(st)
