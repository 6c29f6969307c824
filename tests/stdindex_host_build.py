"""TEST INFRASTRUCTURE: build and bind the host build of the standardized-index device code
(tests/csrc/stdindex_host.cpp over xclim_b200/csrc/stdindex_core.cuh)."""
import ctypes

import numpy as np

import host_build
from xclim_b200 import _lib as L

_vp, _i64, _i32, _f64 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_double
SIGNATURES = {
    "si_host_np_mean": (ctypes.c_float, [_vp, _i32]),
    "si_host_gamma_ml_shape": (_f64, [_f64, _f64, _f64, _vp]),
    "si_host_fit": (_i32, [_vp, _i64, _i64, _vp, _vp, _i32, _i32, _i32, _i32, _f64, _vp, _vp, _vp, _vp]),
    "si_host_apply": (None, [_vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _i32, _i32, _f64, _f64, _f64, _vp]),
}


def load():
    return host_build.load("stdindex", "stdindex_host.cpp", signatures=SIGNATURES)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _vec(name, *args):
    args = [np.ascontiguousarray(np.broadcast_to(a, np.broadcast_shapes(*[np.shape(b) for b in args])),
                                 dtype=np.float64) for a in args]
    out = np.empty(args[0].shape)
    getattr(load(), name)(*[_p(a) for a in args], _i64(out.size), _p(out))
    return out


def gammainc(a, x):
    return _vec("si_host_gammainc", a, x)


def digamma(x):
    return _vec("si_host_digamma", x)


def ndtri(p):
    return _vec("si_host_ndtri", p)


def ndtr(z):
    return _vec("si_host_ndtr", z)


def np_mean(v):
    v = np.ascontiguousarray(v, dtype=np.float32)
    return np.float32(load().si_host_np_mean(_p(v), v.size))


def gamma_ml_shape(s, xa, xb):
    st = np.zeros(1, np.int32)
    a = load().si_host_gamma_ml_shape(float(s), float(xa), float(xb), _p(st))
    return a, int(st[0])


def csr(group_of_step, G, cal=slice(None)):
    """(group_offsets, steps) of the steps in ``cal`` with a group >= 0, steps in time order."""
    gos = np.asarray(group_of_step)
    idx = np.arange(gos.size)[cal]
    g = gos[cal]
    keep = g >= 0
    idx, g = idx[keep], g[keep]
    order = np.argsort(g, kind="stable")
    counts = np.bincount(g, minlength=G)
    return np.concatenate([[0], np.cumsum(counts)]).astype(np.int32), idx[order].astype(np.int32)


def fit(y, group_of_step, G, dist, method, zero_inflated, floc, cal=slice(None)):
    y = np.ascontiguousarray(y, dtype=np.float32)
    T, C = y.shape
    goff, steps = csr(group_of_step, G, cal)
    max_n = max(1, int(np.diff(goff).max()))
    params = np.empty((G, 3, C))
    nz = np.full((G, C), -1, np.int32)
    nn = np.full((G, C), -1, np.int32)
    ws = np.empty(max_n * C, np.float32)
    st = load().si_host_fit(_p(y), C, C, _p(goff), _p(steps), G, L.SI_DISTS[dist], L.SI_METHODS[method],
                            int(zero_inflated), float(floc), _p(params), _p(nz), _p(nn), _p(ws))
    return params, (nz if zero_inflated else None), (nn if zero_inflated else None), st


def apply(y, group_of_step, params, dist, n_zeros=None, n_notnull=None, interp=1.0, alpha=0.0, beta=1.0):
    y = np.ascontiguousarray(y, dtype=np.float32)
    T, C = y.shape
    gos = np.ascontiguousarray(group_of_step, dtype=np.int16)
    params = np.ascontiguousarray(params, dtype=np.float64)
    zi = n_zeros is not None
    nz = np.ascontiguousarray(n_zeros if zi else np.zeros(1), dtype=np.int32)
    nn = np.ascontiguousarray(n_notnull if zi else np.zeros(1), dtype=np.int32)
    out = np.empty((T, C))
    load().si_host_apply(_p(y), T, C, C, _p(gos), _p(params), _p(nz), _p(nn), L.SI_DISTS[dist], int(zi), float(interp),
                         float(alpha), float(beta), _p(out))
    return out
