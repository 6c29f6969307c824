"""TEST INFRASTRUCTURE: build and bind the host build of the ensemble robustness device code
(tests/csrc/ensemble_host.cpp over xclim_b200/csrc/ensemble_core.cuh)."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
_lib = None
_vp, _i64, _i32, _f64 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_double


def load():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.gettempdir(), f"libxclim_b200_ensemble_host_{os.getuid()}.so")
        src = os.path.join(HERE, "csrc", "ensemble_host.cpp")
        csrc = os.path.join(ROOT, "xclim_b200", "csrc")
        deps = [src, os.path.join(csrc, "ensemble_core.cuh"), os.path.join(csrc, "stdindex_core.cuh"),
                os.path.join(csrc, "npsum.cuh"), os.path.join(ROOT, "include", "xclim_b200.h")]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
            tmp = out + f".{os.getpid()}.tmp"
            cmd = ["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", src, "-o", tmp]
            subprocess.run(cmd, check=True, capture_output=True, text=True)
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        lib.ens_host_stdtr.argtypes = [_vp, _vp, _i64, _vp]
        lib.ens_host_ttest_1samp_p.restype = _f64
        lib.ens_host_ttest_1samp_p.argtypes = [_i32, _f64, _f64, _f64]
        lib.ens_host_welch_ttest_p.restype = _f64
        lib.ens_host_welch_ttest_p.argtypes = [_i32, _f64, _f64, _i32, _f64, _f64]
        _lib = lib
    return _lib


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
