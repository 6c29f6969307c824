"""Rain season on the CPU: the oracle against the reference's known answers, the host build of the kernel's scan
against the oracle on seeded series, the host layer over an oracle-backed stand-in, every error, and the argument
checks of the C entry point."""
import ctypes as C
import inspect

import numpy as np
import pytest

import fake_rain_season
import rain_season_cases as cases
import rain_season_host_build as H
from oracle import rain_season_oracle as R
from xb_helpers import make_field
from xclim_b200 import _lib
from xclim_b200.timeaxis import TimeAxis

KNOWN = {"season_found": [3, 100, 97], "start_cond1_fails": [np.nan] * 3, "start_cond2_fails": [np.nan] * 3,
         "end_cond_fails": [3, np.nan, 363]}


def known_series(result_type):
    """tests/test_indices.py:3686-3723 of the reference: NaN except on the set days, in mm/d."""
    x = np.full(365, np.nan, np.float32)
    x[0:3] = 10
    x[3:33] = 5
    x[99:119] = 0
    if result_type == "start_cond1_fails":
        x[2] = 0
    elif result_type == "start_cond2_fails":
        x[10:17] = 0
    elif result_type == "end_cond_fails":
        x[118] = 5
    return x


KNOWN_KW = dict(date_min_start="01-01", date_min_end="01-01")


def host_build(x, ta, freq, scale, params):
    """Start and end steps (float64, NaN for none) of the host build, on the mask the host layer builds."""
    from xclim_b200.indices import _rain_season_mask
    p = {**R.DEFAULTS, **params}
    poff = ta.period_offsets(freq)
    mask = _rain_season_mask(ta, poff, p["date_min_start"], p["date_max_start"], p["date_min_end"], p["date_max_end"])
    s, e = H.rain_season(x, poff, mask, scale, p["thresh_wet_start"], p["window_wet_start"], p["window_not_dry_start"],
                         p["thresh_dry_start"], p["window_dry_start"], _lib.RS_METHODS[p["method_dry_start"]],
                         p["thresh_dry_end"], p["window_dry_end"], _lib.RS_METHODS[p["method_dry_end"]])
    return np.where(s < 0, np.nan, s), np.where(e < 0, np.nan, e)


@pytest.fixture(params=["oracle-on-cpu", pytest.param("cuda", marks=pytest.mark.gpu)])
def backend(request, monkeypatch):
    if request.param == "cuda":
        import torch
        if not torch.cuda.is_available():
            pytest.skip("no CUDA device")
    else:
        fake_rain_season.install(monkeypatch)
    return request.param


# ------------------------------------------------------------------ known answers
@pytest.mark.parametrize("method_dry_start", ["per_day", "total"])
@pytest.mark.parametrize("result_type", list(KNOWN))
def test_known_answers_oracle_and_host_build(result_type, method_dry_start):
    ta = TimeAxis.daily("2000-01-01", 365, "standard")
    x = known_series(result_type)[:, None]
    o = R.rain_season(x, ta, method_dry_start=method_dry_start, **KNOWN_KW)
    np.testing.assert_array_equal([o[k][0, 0] for k in ("start", "end", "length")], KNOWN[result_type])
    s, e = host_build(x, ta, "YS-JAN", 1.0, dict(method_dry_start=method_dry_start, **KNOWN_KW))
    np.testing.assert_array_equal(s, o["start_idx"])
    np.testing.assert_array_equal(e, o["end_idx"])


@pytest.mark.parametrize("method_dry_start", ["per_day", "total"])
@pytest.mark.parametrize("result_type", list(KNOWN))
def test_known_answers_host_layer(backend, result_type, method_dry_start):
    from xclim_b200 import indices
    pr = make_field(known_series(result_type)[:, None], "2000-01-01", "standard", units="mm/d")
    out = indices.rain_season(pr, method_dry_start=method_dry_start, **KNOWN_KW)
    np.testing.assert_array_equal([np.asarray(o.values)[0, 0] for o in out], KNOWN[result_type])
    start, end, length = out
    assert start.name == "rain_season_start" and end.name == "rain_season_end" and length.name == "rain_season_length"
    for o in (start, end):
        assert o.attrs["units"] == "" and o.attrs["is_dayofyear"] == 1 and o.attrs["calendar"] == "standard"
    assert length.attrs["units"] == "days"
    assert all(np.asarray(o.values).dtype == np.float64 for o in out)


# ------------------------------------------------------------------ the host build of the scan against the oracle
@pytest.mark.parametrize("method", ["per_day", "total"])
def test_host_build_matches_oracle(method):
    n_series = 0
    n_start = n_end = 0
    for x, ta, freq, scale, params in cases.cases(11 if method == "per_day" else 12, method, 96):
        try:
            o = R.rain_season(x, ta, freq, scale, **params)
        except ValueError:      # a date window that selects nothing: the host layer raises as well
            with pytest.raises(ValueError, match="select no day"):
                host_build(x, ta, freq, scale, params)
            continue
        s, e = host_build(x, ta, freq, scale, params)
        np.testing.assert_array_equal(s, o["start_idx"], err_msg=str(params))
        np.testing.assert_array_equal(e, o["end_idx"], err_msg=str(params))
        n_series += s.size
        n_start += int(np.isfinite(s).sum())
        n_end += int(np.isfinite(e).sum())
    assert n_series >= 20000
    assert n_start > n_series // 10 and n_end > n_series // 20     # the seasons are not all missing


def test_edge_patterns_match_oracle():
    """Hand-made periods: a start on the last step (the reference indexes past the period there), dry runs that
    straddle the start, an all-dry `total` end window, a single-day S, a truncated last period whose last day
    comes before date_min_start."""
    ta = TimeAxis.daily("2001-01-01", 365 + 100, "noleap")       # the second period ends on 04-10
    T = len(ta)
    x = np.full((T, 6), 5.0, np.float32)
    x[:, 0] = 0
    x[364, 0] = 30                                               # wet on the last day only, N = 1
    x[150:160, 1] = 0                                            # a dry run around the start
    x[158:161, 1] = 9
    x[200:, 2] = 0                                               # dry to the end: all of S_end qualifies
    x[:, 3] = 0
    x[40:50, 3] = 20
    x[:, 5] = np.nan
    cfgs = [dict(window_wet_start=1, window_not_dry_start=0, thresh_wet_start=25.0, date_min_start="01-01",
                 date_min_end="01-01"),
            dict(window_wet_start=2, window_not_dry_start=2, date_min_start="03-01", method_dry_start="total",
                 window_dry_start=3, method_dry_end="total", window_dry_end=5, date_min_end="10-01",
                 date_max_end="04-01"),
            dict(date_min_start="02-09", date_max_start="02-09", thresh_wet_start=20.0, window_wet_start=1,
                 window_not_dry_start=3, date_min_end="02-01"),
            dict(date_min_start="05-01", date_max_start="03-31", date_min_end="01-01", date_max_end="12-31",
                 method_dry_end="total", window_dry_end=1, thresh_dry_end=5.0)]
    for params in cfgs:
        o = R.rain_season(x, ta, "YS", 1.0, **params)
        s, e = host_build(x, ta, "YS", 1.0, params)
        np.testing.assert_array_equal(s, o["start_idx"], err_msg=str(params))
        np.testing.assert_array_equal(e, o["end_idx"], err_msg=str(params))
    o = R.rain_season(x, ta, "YS", 1.0, **cfgs[0])
    assert o["start_idx"][0, 0] == 364 and np.isnan(o["end_idx"][0, 0]) and o["length"][0, 0] == 1
    # a start, then a dry tail that fills every `total` end window of S_end: argmax == argmin, no end
    one = TimeAxis.daily("2001-01-01", 365, "noleap")
    params = dict(thresh_wet_start=15.0, window_not_dry_start=3, date_min_start="05-01", method_dry_end="total",
                  window_dry_end=1, thresh_dry_end=4.75)
    o = R.rain_season(x[:365], one, "YS", 1.0, **params)
    assert o["start_idx"][0, 2] == 122 and np.isnan(o["end_idx"][0, 2]) and o["length"][0, 2] == 365 - 122
    s, e = host_build(x[:365], one, "YS", 1.0, params)
    np.testing.assert_array_equal(s, o["start_idx"])
    np.testing.assert_array_equal(e, o["end_idx"])


# ------------------------------------------------------------------ the host layer over the oracle-backed stand-in
@pytest.mark.parametrize("calendar", ["noleap", "360_day", "standard"])
@pytest.mark.parametrize("freq", ["YS-JAN", "YS-JUL"])
@pytest.mark.parametrize("units", ["mm/d", "kg m-2 s-1"])
def test_host_layer_matches_oracle(backend, calendar, freq, units):
    from xclim_b200 import indices
    scale = 1.0 if units == "mm/d" else 86400.0
    x, ta, _, _, params = next(cases.cases(5, "per_day", 1))
    params = dict(params, date_min_start="04-01", date_max_start="10-31", date_min_end="08-01", date_max_end="06-30")
    ta = TimeAxis.daily("1999-03-01", 1000, calendar)
    x = cases.series(np.random.default_rng(3), 1000, 24, params, scale).reshape(1000, 4, 6)
    pr = make_field(x, "1999-03-01", calendar, units=units)
    start, end, length = indices.rain_season(pr, freq=freq, **{k: (f"{v} mm" if k.startswith("thresh") else v)
                                                               for k, v in params.items()})
    o = R.rain_season(x.reshape(1000, 24), ta, freq, scale, **params)
    for got, key in ((start, "start"), (end, "end"), (length, "length")):
        np.testing.assert_array_equal(np.asarray(got.values).reshape(o[key].shape), o[key])
    assert np.asarray(start.values).shape == (len(ta.period_offsets(freq)) - 1, 4, 6)


def test_signature_follows_the_reference():
    from xclim_b200 import indices
    sig = inspect.signature(indices.rain_season)
    assert list(sig.parameters) == ["pr", "thresh_wet_start", "window_wet_start", "window_not_dry_start",
                                    "thresh_dry_start", "window_dry_start", "method_dry_start", "date_min_start",
                                    "date_max_start", "thresh_dry_end", "window_dry_end", "method_dry_end",
                                    "date_min_end", "date_max_end", "freq"]
    assert {k: p.default for k, p in sig.parameters.items() if k != "pr"} == {
        **{k: (f"{v} mm" if k.startswith("thresh") else v) for k, v in R.DEFAULTS.items()}, "freq": "YS-JAN"}


def test_errors(monkeypatch):
    fake_rain_season.install(monkeypatch)
    from xclim_b200 import indices
    pr = make_field(np.zeros((365, 2), np.float32), "2001-01-01", calendar="noleap", units="mm/d")
    with pytest.raises(ValueError, match=r"Unknown method_dry_start: daily\."):
        indices.rain_season(pr, method_dry_start="daily")
    with pytest.raises(ValueError, match=r"Unknown method_dry_end: sum\."):
        indices.rain_season(pr, method_dry_end="sum")
    for kw in (dict(window_wet_start=0), dict(window_dry_start=0), dict(window_dry_end=0),
               dict(window_not_dry_start=-1), dict(window_wet_start=2.5)):
        with pytest.raises(ValueError, match="must be an integer"):
            indices.rain_season(pr, **kw)
    for kw in (dict(date_min_start="5-01"), dict(date_max_start="13-01"), dict(date_min_end="09/01"),
               dict(date_max_end=1231)):
        with pytest.raises(ValueError, match="MM-DD"):
            indices.rain_season(pr, **kw)
    with pytest.raises(NotImplementedError, match="64"):
        indices.rain_season(pr, window_dry_start=65)
    indices.rain_season(pr, window_dry_start=64, window_dry_end=200, window_wet_start=100)
    # the end window selects no day of the truncated first period (2001-10-01 .. 2001-12-31 with YS)
    short = make_field(np.zeros((200, 2), np.float32), "2001-10-01", calendar="noleap", units="mm/d")
    with pytest.raises(ValueError, match="select no day"):
        indices.rain_season(short, date_min_start="01-01", date_max_start="06-30")
    with pytest.raises(ValueError):
        indices.rain_season(make_field(np.zeros((365, 2), np.float32), "2001-01-01", "noleap", units="mm"))


def test_indicator_masks_missing_periods(monkeypatch):
    """atmos.rain_season is built on first use and masks all three outputs with MissingAny."""
    fake_rain_season.install(monkeypatch)
    from xclim_b200 import atmos
    x = np.stack([known_series("season_found")] * 3, axis=1)
    x[np.isnan(x)] = 2.0
    x[200, 1] = np.nan
    pr = make_field(x, "2001-01-01", calendar="noleap", units="mm/d")
    out = atmos.rain_season(pr, **KNOWN_KW)
    assert len(out) == 3
    for o in out:
        v = np.asarray(o.values)
        assert np.isnan(v[0, 1]) and not np.isnan(v[0, 0]) and v[0, 0] == v[0, 2]


# ------------------------------------------------------------------ the C entry point checks its arguments
@pytest.fixture(scope="module")
def lib():
    import os

    from xclim_b200 import _build
    if not os.path.exists(_build.LIB_PATH):
        _build.build()
    return _lib.load()


def test_entry_point_validates_on_the_host(lib):
    buf = (C.c_float * 64)()
    ibuf = (C.c_int32 * 16)(0, 4)
    mbuf = (C.c_uint8 * 16)()
    p, ip, mp = (C.cast(b, C.c_void_p) for b in (buf, ibuf, mbuf))

    def call(*, x=p, T=4, Cn=4, ldx=4, poff=ip, P=1, mask=mp, ww=3, wnd=30, wds=7, mds=0, wde=20, mde=0, out=p):
        return lib.xc_rain_season_f32(x, T, Cn, ldx, poff, P, mask, 1.0, 25.0, ww, wnd, 1.0, wds, mds, 0.0, wde, mde,
                                      out, p, None)

    INVALID, UNSUPPORTED = _lib.XC_ERR_INVALID, _lib.XC_ERR_UNSUPPORTED
    for kw in (dict(x=None), dict(poff=None), dict(mask=None), dict(out=None)):
        assert call(**kw) == INVALID
        assert b"null pointer" in lib.xc_last_error()
    for kw in (dict(T=0), dict(Cn=0), dict(ldx=3), dict(P=0), dict(P=70000)):
        assert call(**kw) == INVALID
        assert b"shape" in lib.xc_last_error()
    assert call(mds=2) == INVALID and b"method_dry_start" in lib.xc_last_error()
    assert call(mde=-1) == INVALID and b"method_dry_end" in lib.xc_last_error()
    for kw in (dict(ww=0), dict(wds=0), dict(wde=0)):
        assert call(**kw) == INVALID and b"windows" in lib.xc_last_error()
    assert call(wnd=-1) == INVALID and b"window_not_dry_start" in lib.xc_last_error()
    assert call(wds=65) == UNSUPPORTED and b"64" in lib.xc_last_error()
    with pytest.raises(NotImplementedError):
        H.rain_season(np.zeros((4, 4), np.float32), [0, 4], np.zeros(4, np.uint8), 1.0, 25.0, 3, 30, 1.0, 65, 0, 0.0,
                      20, 0)
