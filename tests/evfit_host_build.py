"""TEST INFRASTRUCTURE: build and bind the host build of the frequency-analysis device code
(tests/csrc/evfit_host.cpp over xclim_b200/csrc/evfit_core.cuh)."""
import ctypes

import numpy as np

import host_build
from xclim_b200 import _lib as L

_vp, _i64, _i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32
SIGNATURES = {
    "ev_host_fit": (_i32, [_vp, _i64, _i64, _i64, _i32, _vp, _vp]),
    "ev_host_transform": (None, [_vp, _i64, _i32, _i32, _vp, _i32, _vp]),
    "ev_host_gev_derivs": (None, [_vp, _i32, _vp, _vp, _vp]),
}


def load():
    return host_build.load("evfit", "evfit_host.cpp", signatures=SIGNATURES)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def fit(x, dist):
    """(T, C) float32 -> ((2 | 3, C) float64 params, status) through the host build of fit_cell."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    T, C = x.shape
    params = np.empty((3 if dist == "genextreme" else 2, C))
    ws = np.empty(T * C, np.float32)
    st = load().ev_host_fit(_p(x), T, C, C, L.EV_DISTS[dist], _p(params), _p(ws))
    return params, int(st)


def transform(params, dist, kind, q):
    params = np.ascontiguousarray(params, dtype=np.float64)
    q = np.ascontiguousarray(np.atleast_1d(q), dtype=np.float64)
    C = params.shape[1]
    out = np.empty((q.size, C))
    load().ev_host_transform(_p(params), C, L.EV_DISTS[dist], L.EV_KINDS[kind], _p(q), q.size, _p(out))
    return out


def gev_derivs(x, theta):
    x = np.ascontiguousarray(x, dtype=np.float32)
    th = np.ascontiguousarray(theta, dtype=np.float64)
    g, H = np.empty(3), np.empty(9)
    load().ev_host_gev_derivs(_p(x), x.size, _p(th), _p(g), _p(H))
    return g, H.reshape(3, 3)
