"""The C-ABI library loads and exports every symbol declared in include/xclim_b200.h (no GPU)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "xclim_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(xc_[a-z0-9_]+)\s*\(", src)))


@pytest.fixture(scope="module")
def lib():
    from xclim_b200 import _build, _lib
    if not os.path.exists(_build.LIB_PATH):
        _build.build()
    return _lib.load()


def test_header_symbols_are_exported_and_bound(lib):
    from xclim_b200 import _lib
    syms = declared_symbols()
    assert len(syms) >= 15
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/xclim_b200.h but not exported"
        assert s in _lib.SIGNATURES, f"{s} has no ctypes signature in xclim_b200/_lib.py"
    assert set(_lib.SIGNATURES) == set(syms)


def test_version_and_error_text(lib):
    assert lib.xc_version() == 100
    assert isinstance(lib.xc_last_error(), bytes)


def test_operator_validation_matches_reference_messages():
    # indices/generic.py:285, 296
    from xclim_b200 import _lib
    with pytest.raises(ValueError, match="not recognized"):
        _lib.op_code("=>")
    with pytest.raises(ValueError, match="not permitted"):
        _lib.op_code("==", constrain=(">", "<"))
    assert _lib.op_code("lt") == _lib.op_code("<")


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from xclim_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.XclimB200Error, match="no CPU fallback"):
        _lib.load()


def test_argument_validation_happens_before_any_device_work(lib):
    """Every entry point validates pointers / shapes / enums on the host and reports through the status
    code + xc_last_error() (thread-local) without touching the GPU: checkable on a CPU-only box."""
    import ctypes as C
    from xclim_b200 import _lib
    INVALID, UNSUPPORTED = -1, -2
    buf = (C.c_float * 16)()
    ibuf = (C.c_int32 * 16)()
    p, ip = C.cast(buf, C.c_void_p), C.cast(ibuf, C.c_void_p)
    # null pointers
    assert lib.xc_period_count_f32(None, 4, 4, 4, ip, 1, 0, 0.0, 0, ip, None, None) == INVALID
    assert b"null pointer" in lib.xc_last_error()
    # ldx < C
    assert lib.xc_period_count_f32(p, 4, 4, 2, ip, 1, 0, 0.0, 0, ip, None, None) == INVALID
    assert b"shape" in lib.xc_last_error()
    # unknown operator: the reference's message (indices/generic.py:285)
    assert lib.xc_period_runstat_f32(p, 4, 4, 4, ip, 1, 17, 0.0, 0, 0, 1, 1, p, None, None) == INVALID
    assert b"not recognized" in lib.xc_last_error()
    # window < 1
    assert lib.xc_period_runstat_f32(p, 4, 4, 4, ip, 1, 0, 0.0, 0, 0, 0, 1, p, None, None) == INVALID
    # rolling: unknown window statistic, even centred window
    assert lib.xc_rolling_period_reduce_f32(p, 4, 4, 4, ip, 1, 3, 99, 0, 0, p, None) == INVALID
    assert lib.xc_rolling_period_reduce_f32(p, 8, 4, 4, ip, 1, 4, _lib.STATS["sum"], 1, 0, p, None) == UNSUPPORTED
    assert b"even" in lib.xc_last_error()
    # percentile_doy: even window is unsupported, percentile outside [0, 100] invalid
    doy = (C.c_int16 * 4)(1, 2, 3, 4)
    yr = (C.c_int16 * 4)(0, 0, 0, 0)
    per = (C.c_double * 1)(90.0)
    args = [p, 4, 4, 4, C.cast(doy, C.c_void_p), C.cast(yr, C.c_void_p), 4, 1]
    assert lib.xc_percentile_doy_f32(*args, 4, C.cast(per, C.c_void_p), 1, 1 / 3, 1 / 3, p, p, 64, None) == UNSUPPORTED
    bad = (C.c_double * 1)(101.0)
    assert lib.xc_percentile_doy_f32(*args, 1, C.cast(bad, C.c_void_p), 1, 1 / 3, 1 / 3, p, p, 1024, None) == INVALID
    assert b"[0, 100]" in lib.xc_last_error()
    # eqm: too many quantiles / bad kind
    assert lib.xc_eqm_train_f32(p, p, 4, 4, 4, 65, 0, p, p, None, 0, None) == INVALID
    assert lib.xc_eqm_train_f32(p, p, 4, 4, 4, 20, 7, p, p, None, 0, None) == INVALID
    # the error text is per thread: another thread sees its own (empty) message
    import threading
    seen = []
    th = threading.Thread(target=lambda: seen.append(lib.xc_last_error()))
    th.start(); th.join()
    assert seen == [b""]


def test_boundary_run_entry_points_validate_on_the_host(lib):
    """xc_period_boundary_run_f32, xc_period_boundary_run_range_f32 and xc_period_run_quantile_f32 refuse null
    pointers, P = 0, P > 65535, ldx < C, window 0, q outside [0, 1] and periods too long for the run list before any
    device work."""
    import ctypes as C
    INVALID, UNSUPPORTED = -1, -2
    buf = (C.c_float * 16)()
    p = C.cast(buf, C.c_void_p)
    offs = (C.c_int32 * 3)(0, 4, 8)
    ip = C.cast(offs, C.c_void_p)

    def run(x=p, T=8, Cn=4, ldx=4, poff=ip, P=2, window=1, out=p):
        return lib.xc_period_boundary_run_f32(x, T, Cn, ldx, poff, P, 0, 0.0, 0, window, 0, out, None)

    def rng_(x=p, T=8, Cn=4, ldx=4, poff=ip, lo=ip, hi=ip, P=2, window=1, out=p):
        return lib.xc_period_boundary_run_range_f32(x, T, Cn, ldx, poff, lo, hi, P, 0, 0.0, 0, 0, window, 0, None,
                                                    out, None)

    def rq(x=p, T=8, Cn=4, ldx=4, poff=ip, ph=ip, P=2, q=0.5, window=1, out=p):
        return lib.xc_period_run_quantile_f32(x, T, Cn, ldx, poff, ph, P, 0, 0.0, 0, q, window, 1, out, None)

    for fn in (run, rng_, rq):
        for kw in ({"x": None}, {"poff": None}, {"out": None}):
            assert fn(**kw) == INVALID and b"null pointer" in lib.xc_last_error(), (fn.__name__, kw)
        for kw in ({"P": 0}, {"P": 65536}, {"ldx": 3}, {"T": 0}):
            assert fn(**kw) == INVALID and b"bad shape" in lib.xc_last_error(), (fn.__name__, kw)
        assert fn(window=0) == INVALID and b"window" in lib.xc_last_error(), fn.__name__
    assert rng_(lo=None) == INVALID and rng_(hi=None) == INVALID
    assert rq(ph=None) == INVALID and b"null pointer" in lib.xc_last_error()
    for q in (-1e-9, 1.0 + 1e-9, float("nan")):
        assert rq(q=q) == INVALID and b"q in [0, 1]" in lib.xc_last_error(), q
    # the run list is cap = len / 2 + 2 uint16 per lane, 128 lanes, at most 200 KiB of shared memory
    first_rejected = next(L for L in range(1, 4000) if (L // 2 + 2) * 128 * 2 > 200 * 1024)
    long = (C.c_int32 * 3)(0, 1, 1 + first_rejected)
    assert rq(T=1 + first_rejected, ph=C.cast(long, C.c_void_p)) == UNSUPPORTED
    assert f"periods of {first_rejected} steps".encode() in lib.xc_last_error()


def test_fire_weather_argument_validation(lib):
    """xc_fwi_f32 / xc_fwi_elementwise_f32 refuse inconsistent arguments on the host, with the reference's
    message where it has one (indices/fire/_cffwis.py:1115-1117)."""
    import ctypes as C

    from xclim_b200 import _lib, device
    from xclim_b200.fire import default_params
    INVALID = -1
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    month = C.cast((C.c_int8 * 4)(1, 1, 1, 1), C.c_void_p)
    kw = {k: (v if not isinstance(v, tuple) else v[0]) for k, v in default_params.items()}

    def call(P, tas=p, pr=p, hurs=None, ws=None, snd=None, mask=None, mth=month, lat=p, outs=(p,) + (None,) * 6):
        return lib.xc_fwi_f32(tas, pr, hurs, ws, snd, mask, mth, lat, None, None, None, None, 4, 4, 4, C.byref(P), *outs,
                              None, None, None)

    P = device.fwi_params(None, False, None, True, **kw)
    assert call(P, mth=None) == INVALID and b"month" in lib.xc_last_error()
    assert call(P, outs=(None,) * 7) == INVALID and b"no output" in lib.xc_last_error()
    assert call(P, outs=(None, p) + (None,) * 5) == INVALID and b"hurs" in lib.xc_last_error()      # DMC without hurs
    assert call(P, lat=None) == INVALID and b"lat" in lib.xc_last_error()
    assert call(device.fwi_params(None, True, None, True, **kw)) == INVALID
    assert b"either `season_method` or `season_mask` must be given" in lib.xc_last_error()
    assert call(device.fwi_params("mask", False, None, True, **kw)) == INVALID and b"season_mask" in lib.xc_last_error()
    assert call(device.fwi_params("LA08", False, None, True, **kw)) == INVALID and b"snd" in lib.xc_last_error()
    assert call(device.fwi_params("WF93", False, None, True, **{**kw, "temp_condition_days": 33})) == INVALID
    assert lib.xc_fwi_elementwise_f32(9, p, p, 4, 0.0, 0.0, 0.0, p, None) == INVALID
    assert lib.xc_fwi_elementwise_f32(_lib.FWI_ELEMENTWISE["BUI"], p, None, 4, 0.0, 0.0, 0.0, p, None) == INVALID
