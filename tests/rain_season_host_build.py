"""TEST INFRASTRUCTURE: build and bind the host build of the rain-season scan (tests/csrc/rain_season_host.cpp over
xclim_b200/csrc/rain_season_core.cuh), behind the argument list of device.rain_season with numpy arrays in place of
device tensors."""
import ctypes

import numpy as np

import host_build

_vp, _i64, _i32, _f32, _f64 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_float, ctypes.c_double
SIGNATURES = {
    "rain_season_host": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _vp, _f32, _f64, _i32, _i32, _f64, _i32, _i32, _f64,
                                _i32, _i32, _vp, _vp, ctypes.POINTER(ctypes.c_char_p)]),
}


def load():
    return host_build.load("rain_season", "rain_season_host.cpp", signatures=SIGNATURES)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def rain_season(x2d, poff, mask, scale, thr_wet, window_wet, window_not_dry, thr_dry_start, window_dry_start,
                method_dry_start, thr_dry_end, window_dry_end, method_dry_end, C=None):
    """(start, end) int32 (P, C) steps inside each period, -1 for none.  ``x2d``: (T, ldx) float32 of which the
    first ``C`` columns (all by default) are the cells.  Raises ValueError / NotImplementedError where the C ABI
    returns XC_ERR_INVALID / XC_ERR_UNSUPPORTED."""
    x = np.ascontiguousarray(x2d, dtype=np.float32)
    T, row = x.shape
    C = row if C is None else C
    poff = np.ascontiguousarray(poff, np.int32)
    mask = np.ascontiguousarray(mask, np.uint8)
    P = poff.size - 1
    start = np.full((max(P, 1), C), -2, np.int32)
    end = np.full((max(P, 1), C), -2, np.int32)
    msg = ctypes.c_char_p()
    st = load().rain_season_host(_p(x), T, C, row, _p(poff), P, _p(mask), scale, thr_wet, window_wet,
                                 window_not_dry, thr_dry_start, window_dry_start, method_dry_start, thr_dry_end,
                                 window_dry_end, method_dry_end, _p(start), _p(end), ctypes.byref(msg))
    if st == -2:
        raise NotImplementedError(msg.value.decode())
    if st:
        raise ValueError(msg.value.decode())
    return start, end
