"""TEST INFRASTRUCTURE: build and bind the host build of the chill code (tests/csrc/chill_host.cpp over
xclim_b200/csrc/chill_core.cuh), behind the argument lists of device.chill_daily / chill_hourly /
hourly_temperature with numpy arrays in place of device tensors."""
import ctypes

import numpy as np

import host_build

_vp, _i64, _i32, _f64 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_double
_msg = ctypes.POINTER(ctypes.c_char_p)
SIGNATURES = {
    "chill_host": (_i32, [_i32, _vp, _vp, _vp, _i32, _i64, _i64, _i64, _i64, _vp, _i32, _vp, _vp, _i32, _vp, _f64, _f64,
                          _f64, _f64, _i32, _vp, _vp, _vp, _msg]),
    "hourly_temperature_host": (_i32, [_vp, _vp, _i64, _i64, _i64, _vp, _i32, _vp, _vp, _msg]),
    "dynamic_trace": (None, [_vp, _i64, _vp, _vp]),
}


def load():
    return host_build.load("chill", "chill_host.cpp", signatures=SIGNATURES)


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _raise(st, msg):
    if st:
        raise ValueError(msg.value.decode())


def chill(poff, mask, to_k, to_c, what, *, tasmin=None, tasmax=None, weights=None, lat_index=None, hourly=None,
          C=None):
    """``(cp, cu, valid)`` (P, C) of the fused path (tasmin / tasmax (T, ldx) float32, weights, lat_index) or of
    the hourly path (``hourly`` (H, ldx) float32 / float64); the first ``C`` columns are the cells."""
    poff = np.ascontiguousarray(poff, np.int32)
    P = poff.size - 1
    mask = None if mask is None else np.ascontiguousarray(mask, np.uint8)
    if hourly is None:
        lo = np.ascontiguousarray(tasmin, np.float32)
        hi = np.ascontiguousarray(tasmax, np.float32)
        T, ldx = lo.shape
        H, kind, x, f64 = 24 * T, 0, None, 0
        w = np.ascontiguousarray(weights, np.float64)
        L = w.shape[1]
        li = np.ascontiguousarray(lat_index, np.int32)
    else:
        x = np.ascontiguousarray(hourly)
        H, ldx = x.shape
        T, kind, lo, hi, w, L, li, f64 = -(-H // 24), 1, None, None, None, 0, None, int(x.dtype == np.float64)
    C = ldx if C is None else C
    cp, cu = np.full((max(P, 1), C), -7.0), np.full((max(P, 1), C), -7.0)
    valid = np.full((max(P, 1), C), -7, np.int32)
    msg = ctypes.c_char_p()
    st = load().chill_host(kind, _p(lo), _p(hi), _p(x), f64, T, H, C, ldx, _p(w), L, _p(li), _p(poff), P, _p(mask),
                           to_k[0], to_k[1], to_c[0], to_c[1], what, _p(cp), _p(cu), _p(valid), ctypes.byref(msg))
    _raise(st, msg)
    return cp, cu, valid


def hourly_temperature(tasmin, tasmax, weights, lat_index, C=None):
    lo = np.ascontiguousarray(tasmin, np.float32)
    hi = np.ascontiguousarray(tasmax, np.float32)
    T, ldx = lo.shape
    C = ldx if C is None else C
    w = np.ascontiguousarray(weights, np.float64)
    li = np.ascontiguousarray(lat_index, np.int32)
    out = np.full((24 * T, C), -7.0)
    msg = ctypes.c_char_p()
    st = load().hourly_temperature_host(_p(lo), _p(hi), T, C, ldx, _p(w), w.shape[1], _p(li), _p(out),
                                        ctypes.byref(msg))
    _raise(st, msg)
    return out


def dynamic_trace(tk):
    tk = np.ascontiguousarray(tk, np.float64)
    E = np.empty_like(tk)
    s = ctypes.c_double()
    load().dynamic_trace(_p(tk), tk.size, _p(E), ctypes.byref(s))
    return s.value, E
