"""TEST INFRASTRUCTURE: build and bind the host build of the ensemble robustness device code
(tests/csrc/ensemble_host.cpp over xclim_b200/csrc/ensemble_core.cuh)."""
import ctypes

import numpy as np

import host_build

_vp, _i64, _i32, _f64 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_double
SIGNATURES = {
    "ens_host_stdtr": (None, [_vp, _vp, _i64, _vp]),
    "ens_host_ttest_1samp_p": (_f64, [_i32, _f64, _f64, _f64]),
    "ens_host_welch_ttest_p": (_f64, [_i32, _f64, _f64, _i32, _f64, _f64]),
}


def load():
    return host_build.load("ensemble", "ensemble_host.cpp", signatures=SIGNATURES)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def stdtr(df, t):
    df, t = np.broadcast_arrays(np.asarray(df, np.float64), np.asarray(t, np.float64))
    df, t = np.ascontiguousarray(df), np.ascontiguousarray(t)
    out = np.empty(df.shape)
    load().ens_host_stdtr(_p(df), _p(t), df.size, _p(out))
    return out


def ttest_1samp_p(n, m, ss, popmean):
    return load().ens_host_ttest_1samp_p(int(n), float(m), float(ss), float(popmean))


def welch_ttest_p(n1, m1, ss1, n2, m2, ss2):
    return load().ens_host_welch_ttest_p(int(n1), float(m1), float(ss1), int(n2), float(m2), float(ss2))
