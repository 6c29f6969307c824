"""The ensemble entry points (include/xclim_b200.h e1) are exported and refuse bad arguments on the host, before
any device work (no GPU needed)."""
import ctypes as C
import os

import pytest

INVALID = -1


@pytest.fixture(scope="module")
def lib():
    from xclim_b200 import _build, _lib
    if not os.path.exists(_build.LIB_PATH):
        _build.build()
    return _lib.load()


def test_ensemble_symbols_are_bound(lib):
    from xclim_b200 import _lib
    for s in ("xc_ens_percentiles_f32", "xc_ens_moments_f32", "xc_ens_robustness_f32"):
        assert hasattr(lib, s) and s in _lib.SIGNATURES


def test_percentiles_and_moments_argument_checks(lib):
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    per = (C.c_double * 33)(*([50.0] * 33))
    pp = C.cast(per, C.c_void_p)

    def perc(x=p, R=4, N=4, ldr=4, per=pp, n=1, a=1.0, b=1.0, mm=1, out=p):
        return lib.xc_ens_percentiles_f32(x, R, N, ldr, per, n, a, b, mm, out, None)

    def mom(x=p, R=4, N=4, ldr=4, mm=1, outs=(p, p, p, p)):
        return lib.xc_ens_moments_f32(x, R, N, ldr, None, mm, *outs, None)

    for fn in (perc, mom):
        assert fn(x=None) == INVALID and b"null pointer" in lib.xc_last_error()
        for R in (0, 129):
            assert fn(R=R) == INVALID and b"1 to 128 members" in lib.xc_last_error(), (fn.__name__, R)
        assert fn(ldr=3) == INVALID and b"bad shape" in lib.xc_last_error()
        assert fn(N=0) == INVALID and b"bad shape" in lib.xc_last_error()
        assert fn(mm=-1) == INVALID and b"min_members" in lib.xc_last_error()
    assert perc(per=None) == INVALID and perc(out=None) == INVALID
    assert perc(n=0) == INVALID and perc(n=33) == INVALID and b"percentiles per call" in lib.xc_last_error()
    bad = (C.c_double * 1)(100.5)
    assert perc(per=C.cast(bad, C.c_void_p)) == INVALID and b"[0, 100]" in lib.xc_last_error()
    assert perc(a=1.5) == INVALID and b"alpha and beta" in lib.xc_last_error()
    assert mom(outs=(p, None, p, p)) == INVALID and b"null pointer" in lib.xc_last_error()


def test_robustness_argument_checks(lib):
    from xclim_b200 import _lib
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    d = C.cast((C.c_double * 8)(), C.c_void_p)
    T = _lib.ENS_TESTS

    def rob(fut=p, Tf=2, lf=(8, 4), ref=p, Tr=2, lr=(8, 4), ann=None, P=0, la=0, ys=None, R=2, Cn=4,
            test=T["ttest"], param=0.05, frac=d, pv=p):
        return lib.xc_ens_robustness_f32(fut, Tf, *lf, ref, Tr, *lr, ann, P, la, ys, R, Cn, None, test, param, 1,
                                         frac, pv, None)

    assert rob(fut=None) == INVALID and rob(frac=None) == INVALID and b"null pointer" in lib.xc_last_error()
    for kw in ({"R": 0}, {"Cn": 0}, {"Tf": 0}, {"lf": (3, 4)}, {"lf": (8, 3)}, {"Tr": 0}, {"lr": (8, 2)}):
        assert rob(**kw) == INVALID and b"bad shape" in lib.xc_last_error(), kw
    assert rob(test=7) == INVALID and b"unknown test" in lib.xc_last_error()
    ipcc = {"test": T["ipcc-ar6-c"], "pv": None}
    for kw in ({}, {"ann": p, "P": 2, "la": 8}, {"ys": d, "P": 2, "la": 8}, {"ann": p, "ys": d, "P": 0, "la": 8},
               {"ann": p, "ys": d, "P": 2, "la": 7}):
        assert rob(**ipcc, **kw) == INVALID and b"annual means" in lib.xc_last_error(), kw
    assert rob(ref=None, pv=None) == INVALID
    assert b"When deltas are given (ref=None), 'test' must be None or 'threshold'." in lib.xc_last_error()
    assert rob(ref=None, test=T["rel_thresh"], pv=None) == INVALID
    assert rob(test=T["abs_thresh"]) == INVALID and b"pvals" in lib.xc_last_error()
    assert rob(param=float("nan")) == INVALID and b"NaN" in lib.xc_last_error()
