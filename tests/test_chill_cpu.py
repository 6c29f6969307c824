"""Chill portions, chill units and the hourly temperature on the CPU: the oracle against the reference's goldens
and known answers, the host build of chill_core.cuh against the oracle, the host layer over CPU stand-ins, every
error, and the argument checks of the C entry points."""
import os

import numpy as np
import pytest

import chill_host_build as H
import fake_chill
from oracle import chill_oracle as O
from xclim_b200 import Field, TimeAxis, _lib, atmos, converters, indices
from xclim_b200.chill import HourlyAxis, HourlyTemperature

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "ref_chill.npz"))
CASES = (("360_day", 360), ("noleap", 365), ("standard", 366))
K2C = 273.15
PORTIONS, UNITS, POS = _lib.CHILL_PORTIONS, _lib.CHILL_UNITS, _lib.CHILL_POSITIVE_ONLY
# the known answer of the reference's tests/test_helpers.py:302-365 (lat 0, tasmin 0 degC, tasmax 20 degC)
KNOWN = [0.0, 3.90180644, 7.65366865, 11.11140466, 14.14213562, 16.62939225, 18.47759065, 19.61570561, 20.0,
         19.61570561, 18.47759065, 16.62939225, 14.14213562, 10.32039099, 8.0848137, 6.49864636, 5.26831939,
         4.26306907, 3.41314202, 2.67690173, 2.02749177, 1.44657476, 0.92107141, 0.44132444]


def _axis(cal, n):
    return TimeAxis.daily(f"{int(GOLD[f'year_{cal}'])}-01-01", n, cal)


def _daylen(cal, n, infill, lats=None):
    ta = _axis(cal, n)
    da = converters.day_angle(ta.year, ta.doy, cal)[:, None]
    return converters.day_lengths(da, (GOLD["lats"] if lats is None else lats)[None, :], infill)


# ------------------------------------------------------------------------------------------ oracle vs reference
@pytest.mark.parametrize("cal,n", CASES)
@pytest.mark.parametrize("infill", [False, True])
def test_oracle_reproduces_reference(cal, n, infill):
    key = f"{cal}_{int(infill)}"
    dl = _daylen(cal, n, infill)
    np.testing.assert_array_equal(dl, GOLD[f"daylen_{key}"])
    hr = O.hourly_temperature(GOLD[f"tasmin_{cal}"], GOLD[f"tasmax_{cal}"], dl)
    keep = (np.arange(24 * n) // 24) % int(GOLD["keep_every"]) == 0
    np.testing.assert_array_equal(hr[keep], GOLD[f"hourly_{key}"])          # bit for bit, NaN where NaN
    for c in range(dl.shape[1]):
        s, E, delta = O.dynamic(hr[:, c] + K2C)
        assert np.sum(delta != 0) == GOLD[f"cp_hours_{key}"][c]
        np.testing.assert_allclose(s, GOLD[f"cp_{key}"][c], rtol=1e-12)


def test_day_lengths_default_unchanged_and_infill():
    ta = _axis("standard", 366)
    da = converters.day_angle(ta.year, ta.doy, "standard")[:, None]
    lats = GOLD["lats"][None, :]
    with np.errstate(invalid="ignore"):
        plain = (24 / np.pi) * np.arccos(-np.tan(lats * (np.pi / 180)) * np.tan(converters.solar_declination(da)))
    np.testing.assert_array_equal(converters.day_lengths(da, lats), plain)
    filled = converters.day_lengths(da, lats, infill_polar_days=True)
    polar = np.isnan(plain) & (np.abs(lats) > 66.5)
    assert polar.any() and not np.isnan(filled[polar]).any()
    assert set(np.unique(filled[polar])) == {0.0, 24.0}


def test_known_answer_oracle():
    dl = converters.day_lengths(converters.day_angle(np.array([2000]), np.array([1]), "standard")[:, None],
                                np.array([[0.0]]))
    hr = O.hourly_temperature(np.array([[0.0]]), np.array([[20.0]]), dl)
    np.testing.assert_allclose(hr[:, 0], KNOWN)


def test_reference_index_known_answers():
    """tests/test_indices.py:375-398 of the reference (hourly series in K)."""
    tas = np.linspace(0, 15, 120 * 24) + K2C
    assert np.round(O.dynamic(tas)[0], 7) == pytest.approx(72.2441765, abs=1e-7)
    tas = np.array(10 * [1.1] + 15 * [2.0] + 20 * [5.6] + 10 * [16.0] + 5 * [20.0]) + K2C
    cp, cu, _ = O.chill(tas[:, None], [0, 3], positive_only=False)
    assert cu[0, 0] == 0.5 * 15 + 20 - 0.5 * 10 - 5
    cp, cu, _ = O.chill(tas[:, None], [0, 3], positive_only=True)
    assert cu[0, 0] == 0.5 * 15 + 20 - 0.5 * 3


# ------------------------------------------------------------------------------------------ host build vs oracle
def _weights(cal, n, infill):
    ta = _axis(cal, n)
    return converters.hourly_weights(ta, GOLD["lats"], infill)


@pytest.mark.parametrize("cal,n", CASES)
@pytest.mark.parametrize("infill", [False, True])
def test_host_build_hours_and_models(cal, n, infill):
    lo, hi = GOLD[f"tasmin_{cal}"], GOLD[f"tasmax_{cal}"]
    L = lo.shape[1]
    w = _weights(cal, n, infill)
    li = np.arange(L, dtype=np.int32)
    hr = H.hourly_temperature(lo, hi, w, li)
    exp = O.hourly_temperature(lo, hi, _daylen(cal, n, infill))
    np.testing.assert_array_equal(hr, exp)
    ta = _axis(cal, n)
    poff = ta.period_offsets("MS")
    mask = ta.select_mask(date_bounds=("02-10", "11-20"))
    for pos in (False, True):
        what = PORTIONS | UNITS | (POS if pos else 0)
        cp, cu, valid = H.chill(poff, mask, (1.0, K2C), (1.0, 0.0), what, tasmin=lo, tasmax=hi, weights=w,
                                lat_index=li)
        cp_h, cu_h, valid_h = H.chill(poff, mask, (1.0, K2C), (1.0, 0.0), what, hourly=exp)
        ocp, ocu, ovalid = O.chill(exp, poff, mask, (1.0, K2C), (1.0, 0.0), positive_only=pos)
        np.testing.assert_array_equal(cu, ocu)
        np.testing.assert_array_equal(valid, ovalid)
        np.testing.assert_allclose(cp, ocp, rtol=1e-11, atol=1e-12)
        for a, b in ((cp, cp_h), (cu, cu_h), (valid, valid_h)):
            np.testing.assert_array_equal(a, b)     # the fused and hourly-input paths on the same hours


def test_host_build_dynamic_trace_counts():
    """The E >= 1 hours of the host build's recurrence are the oracle's, on a season through the threshold."""
    rng = np.random.default_rng(3)
    for n in (1, 2, 500, 3000):
        tk = K2C + rng.uniform(-5, 20, n)
        tk[rng.integers(0, n, max(1, n // 997))] = np.nan if n > 600 else tk[0]
        s, E = H.dynamic_trace(tk)
        so, Eo, _ = O.dynamic(tk)
        np.testing.assert_array_equal(E >= 1, Eo >= 1)
        np.testing.assert_array_equal(np.isnan(E), np.isnan(Eo))
        np.testing.assert_allclose(E, Eo, rtol=1e-12, equal_nan=True)
        np.testing.assert_allclose(s, so, rtol=1e-11)


def test_nan_hour_stops_the_recurrence():
    tk = K2C + np.full(500, 5.0)
    s_full = H.dynamic_trace(tk)[0]
    tk[300] = np.nan
    s, E = H.dynamic_trace(tk)
    assert np.isnan(E[300:]).all() and not np.isnan(E[:300]).any()
    assert s == H.dynamic_trace(tk[:300])[0] and 0 < s < s_full


def test_polar_night_without_infill_gives_no_portions():
    lo = np.full((366, 2), -2.0, np.float32)
    hi = lo + 8
    ta = TimeAxis.daily("2000-01-01", 366, "standard")
    w = converters.hourly_weights(ta, np.array([0.0, 80.0]), False)
    cp, cu, valid = H.chill(np.array([0, 366]), None, (1.0, K2C), (1.0, 0.0), PORTIONS | UNITS, tasmin=lo, tasmax=hi,
                            weights=w, lat_index=np.array([0, 1], np.int32))
    assert valid[0, 1] < valid[0, 0] == 366 * 24
    assert cp[0, 0] > 0 and np.isfinite(cp[0, 1])


# ------------------------------------------------------------------------------------------ host layer
def _field(v, start="2000-01-01", cal="standard", units="degC", dims=("time", "lat"), lat=None, name=None):
    v = np.asarray(v, np.float32)
    coords = {} if lat is None else {"lat": np.asarray(lat, np.float64)}
    return Field(v, dims, TimeAxis.daily(start, v.shape[0], cal), coords, {"units": units}, name)


@pytest.fixture
def fake(monkeypatch):
    fake_chill.install(monkeypatch)


@pytest.mark.parametrize("lat_on", ["tasmin", "both"])
def test_known_answer_host_layer(fake, lat_on):
    """tests/test_helpers.py:302-365: tasmax passed first, merged by name."""
    tasmax = Field(np.array([20.0], np.float32), ("time",), TimeAxis.daily("2000-01-01", 1), {}, {"units": "degC"},
                   "tasmax")
    tasmin = _field([[0.0]], lat=[0.0], name="tasmin")
    if lat_on == "both":
        tasmax = _field([[20.0]], lat=[0.0], name="tasmax")
    h = indices.make_hourly_temperature(tasmax, tasmin)
    assert isinstance(h, HourlyTemperature) and h.attrs["units"] == "degC" and h.shape == (24, 1)
    np.testing.assert_allclose(np.asarray(h.values)[:, 0], KNOWN)
    assert np.asarray(h.values).dtype == np.float64


def _grid(seed=0, n=3 * 365 + 1, L=4, cal="standard"):
    rng = np.random.default_rng(seed)
    lo = rng.uniform(-10, 12, (n, L)).astype(np.float32)
    hi = (lo + rng.uniform(0, 12, (n, L))).astype(np.float32)
    lo[5, 1] = np.nan
    lats = np.array([-70.0, 10.0, 45.0, 80.0])[:L]
    return _field(lo, cal=cal, lat=lats, name="tasmin"), _field(hi, cal=cal, lat=lats, name="tasmax")


@pytest.mark.parametrize("infill", [False, True])
def test_lazy_equals_materialised(fake, infill):
    lo, hi = _grid()
    h = indices.make_hourly_temperature(lo, hi, infill_polar_days=infill)
    mat = Field(np.asarray(h.values), h.dims, h.time, dict(h.coords), dict(h.attrs))
    dl = converters.day_lengths(converters.day_angle(lo.time.year, lo.time.doy, "standard")[:, None],
                                lo.coords["lat"][None, :], infill)
    np.testing.assert_array_equal(mat.values, O.hourly_temperature(lo.values, hi.values, dl))
    for kw in ({}, {"date_bounds": ("09-01", "03-30"), "freq": "YS-JUL"}):
        a, b = indices.chill_portions(h, **kw), indices.chill_portions(mat, **kw)
        np.testing.assert_array_equal(a.values, b.values)
        np.testing.assert_array_equal(a.coords["time"], b.coords["time"])
    for pos in (False, True):
        a, b = indices.chill_units(h, positive_only=pos), indices.chill_units(mat, positive_only=pos)
        np.testing.assert_array_equal(a.values, b.values)
        o = O.chill(mat.values, lo.time.period_offsets("YS"), positive_only=pos, to_c=(1.0, 0.0))[1]
        np.testing.assert_array_equal(a.values, o)


def test_chill_portions_against_oracle_and_seasons(fake):
    lo, hi = _grid(n=4 * 365 + 1)        # 2000-01-01 .. 2003-12-31
    h = indices.make_hourly_temperature(lo, hi)
    cp = indices.chill_portions(h, date_bounds=("09-01", "03-30"), freq="YS-JUL")
    assert cp.values.shape == (5, 4) and cp.values.dtype == np.float64     # 5 seasons from 4 years
    assert list(cp.coords["time"])[0].startswith("1999-07")
    ta = lo.time
    mask = ta.select_mask(date_bounds=("09-01", "03-30"))
    poff = ta.period_offsets("YS-JUL")
    exp = O.chill(np.asarray(h.values), poff, mask, (1.0, K2C))[0]
    np.testing.assert_allclose(cp.values, exp, rtol=1e-11)
    ind = atmos.chill_portions(h, date_bounds=("09-01", "03-30"), freq="YS-JUL")
    assert ind.name == "cp" and ind.attrs["units"] == "1"
    v = np.asarray(ind.values)
    assert np.isnan(v[0]).all() and np.isnan(v[-1]).all()       # incomplete first and last seasons
    assert np.isnan(v[:, [0, 3]]).all()                          # polar nights without infill: missing hours
    np.testing.assert_array_equal(v[1:-1, 1:3], cp.values[1:-1, 1:3])


def test_indicator_units_mask_and_missing(fake):
    lo, hi = _grid(n=4 * 365 + 1)
    h = indices.make_hourly_temperature(lo, hi)
    cu = atmos.chill_units(h, date_bounds=("04-01", "06-30"))
    assert cu.name == "cu" and cu.attrs["units"] == "1" and cu.values.shape == (4, 4)
    mask = lo.time.select_mask(date_bounds=("04-01", "06-30"))
    exp = O.chill(np.asarray(h.values), lo.time.period_offsets("YS"), mask, to_c=(1.0, 0.0))[1]
    v = np.asarray(cu.values)
    np.testing.assert_array_equal(v[:, 1:3], exp[:, 1:3])
    assert np.isnan(v[:, [0, 3]]).all()      # polar night / day without infill: NaN hours, hence missing


def test_explicit_hourly_input_and_partial_day(fake):
    tas = np.array(10 * [1.1] + 15 * [2.0] + 20 * [5.6] + 10 * [16.0] + 5 * [20.0]) + K2C
    f = Field(tas, ("time",), HourlyAxis.hourly("2000-01-01", tas.size), {}, {"units": "K"})
    assert indices.chill_units(f).values[0] == 0.5 * 15 + 20 - 0.5 * 10 - 5
    assert indices.chill_units(f, positive_only=True).values[0] == 0.5 * 15 + 20 - 0.5 * 3
    f = Field(np.linspace(0, 15, 120 * 24) + K2C, ("time",), HourlyAxis.hourly("2000-01-01", 120 * 24), {},
              {"units": "K"})
    np.testing.assert_allclose(indices.chill_portions(f).values, [72.2441765], atol=1e-7)
    f32 = Field(f.values.astype(np.float32), f.dims, f.time, {}, {"units": "K"})
    np.testing.assert_allclose(indices.chill_portions(f32).values,
                               O.chill(f.values.astype(np.float32)[:, None], [0, 120])[0][0], rtol=1e-12)


def test_errors(fake):
    lo, hi = _grid()
    with pytest.raises(NotImplementedError):
        indices.chill_units(lo)                             # daily data
    with pytest.raises(ValueError, match="units"):
        indices.make_hourly_temperature(lo, Field(hi.values, hi.dims, hi.time, dict(hi.coords), {"units": "K"}))
    with pytest.raises(ValueError, match="latitude"):
        indices.make_hourly_temperature(Field(lo.values, lo.dims, lo.time, {}, {"units": "degC"}),
                                        Field(hi.values, hi.dims, hi.time, {}, {"units": "degC"}))
    h = indices.make_hourly_temperature(lo, hi)
    with pytest.raises(ValueError, match="allowed"):
        atmos.chill_portions(h, freq="MS")
    with pytest.raises(ValueError, match="allowed"):
        atmos.chill_units(h, freq="QS-DEC")
    with pytest.raises(ValueError):
        HourlyAxis(TimeAxis.daily("2000-01-01", 3), 24)
    bad = Field(np.zeros(48), ("time",), HourlyAxis.hourly("2000-01-01", 47), {}, {"units": "K"})
    with pytest.raises(ValueError, match="hourly axis"):
        indices.chill_units(bad)
    with pytest.raises(ValueError, match="selects no day"):
        indices.chill_portions(h, doy_bounds=(400, 400))


def test_c_argument_checks():
    lo = np.zeros((3, 2), np.float32)
    w = np.zeros((3, 1, _lib.CHILL_ROW))
    li = np.zeros(2, np.int32)
    poff = np.array([0, 3], np.int32)
    ok = dict(tasmin=lo, tasmax=lo, weights=w, lat_index=li)
    H.chill(poff, None, (1, 0), (1, 0), PORTIONS, **ok)
    for what in (0, 8, POS):
        with pytest.raises(ValueError, match="output selection"):
            H.chill(poff, None, (1, 0), (1, 0), what, **ok)
    with pytest.raises(ValueError, match="bad shape"):
        H.chill(np.array([0], np.int32), None, (1, 0), (1, 0), PORTIONS, **ok)
    with pytest.raises(ValueError, match="bad shape"):
        H.chill(poff, None, (1, 0), (1, 0), UNITS, **ok, C=3)
    with pytest.raises(ValueError, match="bad shape"):
        H.chill(poff, None, (1, 0), (1, 0), UNITS, **{**ok, "weights": np.zeros((3, 0, _lib.CHILL_ROW))})
    x = np.zeros((49, 2))
    H.chill(poff, None, (1, 0), (1, 0), UNITS, hourly=x)
    with pytest.raises(ValueError, match="bad shape"):
        H.chill(np.array([0, 1], np.int32), None, (1, 0), (1, 0), UNITS, hourly=np.zeros((48, 2)), C=3)
