"""The ETCCDI day-of-year percentile indices (WSDI, CSDI, R95pTOT), the compound percentile days and the daily
temperature range: the oracle against the reference's known answers and hand-built series, the host layer over
oracle-backed stand-ins (and on the GPU through the ``cuda`` backend), and the host-side checks of the C entry
points."""
import ctypes as C
import inspect

import numpy as np
import pytest

import fake_etccdi
from oracle import etccdi_oracle as E
from oracle import xclim_oracle as O
from xb_helpers import make_field


@pytest.fixture(params=["oracle-on-cpu", pytest.param("cuda", marks=pytest.mark.gpu)])
def backend(request, monkeypatch):
    if request.param == "cuda":
        import torch
        if not torch.cuda.is_available():
            pytest.skip("no CUDA device")
    else:
        fake_etccdi.install(monkeypatch)
    return request.param


def _sine_series(bump, sign, seed):
    """tests/test_indices.py:105-115, 3164-3174: ten years of a seasonal sine with a 10-day bump in July 2000."""
    i = 3650
    x = np.zeros(i) + 10.0 * np.sin(np.arange(i) / 365.0 * 2 * np.pi) + 0.1 * np.random.default_rng(seed).random(i)
    x[10:20] += sign * bump
    return x.astype(np.float32)


# ------------------------------------------------------------------ the oracle
def test_oracle_wsdi_csdi_simple():
    """The reference's test_simple of both indices, with the oracle's percentile_doy (366-day table)."""
    from xclim_b200 import TimeAxis
    ta = TimeAxis.daily("2000-07-01", 3650, "standard")
    doy = np.asarray(ta.doy)
    year = np.searchsorted(np.unique(ta.year), ta.year)
    poff = ta.period_offsets("YS")
    tx = _sine_series(2, 1, 1)
    tab = O.percentile_doy(tx[:, None], year, doy, 5, 90.0)[:, 0]
    out = E.warm_spell_duration_index(tx[:, None], tab, doy, poff)
    assert out[0, 0] == 10
    tn = _sine_series(2, -1, 2)
    tab = O.percentile_doy(tn[:, None], year, doy, 5, 10.0)[:, 0]
    out = E.cold_spell_duration_index(tn[:, None], tab, doy, poff)
    assert out[0, 0] == 10


def test_oracle_fraction_over_precip_thresh_by_hand():
    pr = np.zeros((10, 2), np.float32)
    pr[:, 0] = [0, 0.5, 2, 3, 10, 20, np.nan, 1, 1.5, 0]
    pr[:, 1] = [0, 0.5, 0.9, 0, 0, 0, 0, 0, 0, 0]                # no wet day -> 0 / 0
    poff = np.array([0, 5, 10])
    doy = np.arange(1, 11)
    tab = np.full((10, 2), 2.5)
    tab[3, 0] = np.nan                                          # a NaN entry falls back to thresh
    out = E.fraction_over_precip_thresh(pr, tab, 1.0, poff, doy=doy)
    # period 0: wet = 2 + 3 + 10 = 15 (> 1); over tp: 3 (tp -> 1 at doy 4), 10 -> 13
    np.testing.assert_allclose(out[0, 0], np.float32(13) / np.float32(15))
    # period 1: wet = 20 + 1.5 (the NaN day and the day at the threshold are not wet); over: 20
    np.testing.assert_allclose(out[1, 0], np.float32(20) / np.float32(21.5))
    assert np.isnan(out[0, 1]) and np.isnan(out[1, 1])
    # one threshold per cell, lower than thresh -> thresh; ">=" takes the day at the threshold
    per_cell = np.array([0.5, 2.0])
    out = E.fraction_over_precip_thresh(pr, per_cell, 1.0, poff, op=">=")
    np.testing.assert_allclose(out[:, 0], [1, 1])               # tp = thresh: every wet day is over it
    assert np.isnan(out[:, 1]).all()                            # cell 1 has no day >= 1 mm/d


def test_oracle_compound_days_by_hand():
    tas = np.array([[1, 5, 1, 5, 1]], np.float32).T
    pr = np.array([[0, 0, 9, 9, np.nan]], np.float32).T
    tt = np.full((5, 1), 3.0)
    pt = np.full((5, 1), 4.0)
    poff = np.array([0, 5])
    doy = np.arange(1, 6)
    got = {n: E.compound_days(n, tas, pr, tt, pt, doy, poff)[0, 0] for n in E._COMPOUND}
    assert got == {"cold_and_dry_days": 1, "warm_and_dry_days": 1, "warm_and_wet_days": 1, "cold_and_wet_days": 1}


def test_oracle_dtr_by_hand():
    lo = np.array([0, 1, 2, np.nan, 0, 0], np.float32)[:, None]
    hi = np.array([5, 5, 5, 5, 10, 4], np.float32)[:, None]
    poff = np.array([0, 3, 6])
    np.testing.assert_allclose(E.daily_temperature_range(lo, hi, poff, "mean")[:, 0], [4, 7])
    np.testing.assert_allclose(E.daily_temperature_range(lo, hi, poff, "max")[:, 0], [5, 10])
    # d = 5 4 3 nan 10 4: diffs (upper label) nan 1 1 | nan nan 6 -> the second period's first diff crosses the edge
    np.testing.assert_allclose(E.daily_temperature_range_variability(lo, hi, poff)[:, 0], [1, 6])


# ------------------------------------------------------------------ the host layer (CPU stand-ins and the GPU)
def test_wsdi_csdi_simple(backend):
    from xclim_b200 import calendar as xcal
    from xclim_b200 import indices
    tx = make_field(_sine_series(2, 1, 1), "2000-07-01", units="K")
    tx90 = xcal.select_percentile(xcal.percentile_doy(tx, per=90), 90.0)
    out = indices.warm_spell_duration_index(tx, tx90, freq="YS")
    assert out.values[0] == 10 and out.attrs["units"] == "d" and out.values.dtype == np.float32
    tn = make_field(_sine_series(2, -1, 2), "2000-07-01", units="K")
    tn10 = xcal.select_percentile(xcal.percentile_doy(tn, per=10), 10.0)
    out = indices.cold_spell_duration_index(tn, tn10, freq="YS")
    assert out.values[0] == 10 and out.attrs["units"] == "d"
    # the table converted to the data's units first: the same answer from degC data
    tnc = make_field(_sine_series(2, -1, 2) - np.float32(273.15), "2000-07-01", units="degC")
    assert indices.cold_spell_duration_index(tnc, tn10, freq="YS").values[0] == 10


def _per_field(table, units, cell_dims=("d0",)):
    """A (cells, dayofyear) percentile array like percentile_doy's, one percentile selected."""
    from xclim_b200 import Field
    vals = np.ascontiguousarray(np.moveaxis(np.asarray(table, np.float64), 0, -1))
    return Field(vals, cell_dims + ("dayofyear",), None, {"dayofyear": np.arange(1, table.shape[0] + 1)},
                 {"units": units})


def test_fraction_over_precip_thresh_host(backend):
    from xclim_b200 import Field, indices
    rng = np.random.default_rng(3)
    T = 730
    x = (rng.gamma(0.6, 4.0, (T, 3)) * (rng.random((T, 3)) < 0.5)).astype(np.float32)
    x[5, 0] = np.nan
    pr = make_field(x, "2001-01-01", calendar="noleap", units="mm/d")
    tab = rng.gamma(2.0, 3.0, (365, 3))
    tab[10:20, 1] = np.nan
    per = _per_field(tab, "mm/d")
    out = indices.fraction_over_precip_thresh(pr, per, thresh="1 mm/day", freq="YS")
    exp = E.fraction_over_precip_thresh(x, tab, 1.0, np.array([0, 365, 730]), doy=np.asarray(pr.time.doy))
    np.testing.assert_allclose(out.values, exp, rtol=1e-6)
    assert out.attrs["units"] == "" and out.values.dtype == np.float32
    # per-cell thresholds in other units (kg m-2 s-1)
    pc = Field(np.array([3.0, 0.5, 8.0]) / 86400.0, ("d0",), None, {}, {"units": "kg m-2 s-1"})
    out = indices.fraction_over_precip_thresh(pr, pc, thresh="1 mm/day", freq="YS", op=">=")
    exp = E.fraction_over_precip_thresh(x, np.array([3.0, 0.5, 8.0]), 1.0, np.array([0, 365, 730]), op=">=")
    np.testing.assert_allclose(out.values, exp, rtol=1e-5)


@pytest.mark.parametrize("name", sorted(E._COMPOUND))
def test_compound_days_host(backend, name):
    from xclim_b200 import indices
    rng = np.random.default_rng(4)
    T = 365 * 2
    t = (280 + 5 * rng.standard_normal((T, 4))).astype(np.float32)
    p = (rng.gamma(0.7, 3.0, (T, 4))).astype(np.float32)
    t[7, 1] = np.nan
    tas = make_field(t, "2001-01-01", calendar="noleap", units="K")
    pr = make_field(p, "2001-01-01", calendar="noleap", units="mm/d")
    tt = 280 + 2 * rng.standard_normal((365, 4))
    pt = rng.gamma(1.0, 2.0, (365, 4))
    out = getattr(indices, name)(tas, pr, _per_field(tt, "K"), _per_field(pt, "mm/d"), freq="MS")
    exp = E.compound_days(name, t, p, tt, pt, np.asarray(tas.time.doy), tas.time.period_offsets("MS"))
    np.testing.assert_array_equal(out.values, exp)
    assert out.values.dtype == np.int64 and out.attrs["units"] == "d"


@pytest.mark.parametrize("op", ["mean", "min", "max", "std"])
def test_dtr_host(backend, op):
    from xclim_b200 import indices
    rng = np.random.default_rng(5)
    lo = (270 + 5 * rng.standard_normal((400, 3))).astype(np.float32)
    hi = (lo + 8 + 2 * rng.standard_normal((400, 3))).astype(np.float32)
    lo[[0, 31, 32], 1] = np.nan
    a, b = make_field(lo, units="K"), make_field(hi, units="K")
    poff = a.time.period_offsets("MS")
    out = indices.daily_temperature_range(a, b, freq="MS", op=op)
    np.testing.assert_allclose(out.values, E.daily_temperature_range(lo, hi, poff, op), rtol=2e-6, atol=1e-5)
    assert out.attrs["units"] == "K" and out.attrs["units_metadata"] == "temperature: difference"
    if op == "mean":
        v = indices.daily_temperature_range_variability(a, b, freq="MS")
        np.testing.assert_allclose(v.values, E.daily_temperature_range_variability(lo, hi, poff), rtol=2e-6)


def test_signatures_follow_the_reference():
    from xclim_b200 import indices
    want = {
        "warm_spell_duration_index": "(tasmax, tasmax_per, window=6, freq='YS', resample_before_rl=True, "
                                     "bootstrap=False, op='>')",
        "cold_spell_duration_index": "(tasmin, tasmin_per, window=6, freq='YS', resample_before_rl=True, "
                                     "bootstrap=False, op='<')",
        "fraction_over_precip_thresh": "(pr, pr_per, thresh='1 mm/day', freq='YS', bootstrap=False, op='>')",
        "cold_and_dry_days": "(tas, pr, tas_per, pr_per, freq='YS')",
        "warm_and_dry_days": "(tas, pr, tas_per, pr_per, freq='YS')",
        "warm_and_wet_days": "(tas, pr, tas_per, pr_per, freq='YS')",
        "cold_and_wet_days": "(tas, pr, tas_per, pr_per, freq='YS')",
        "daily_temperature_range": "(tasmin, tasmax, freq='YS', op='mean')",
        "daily_temperature_range_variability": "(tasmin, tasmax, freq='YS')",
    }
    for name, sig in want.items():
        fn = getattr(indices, name)
        assert str(inspect.signature(getattr(fn, "__wrapped_index__", fn))) == sig, name


def test_errors(monkeypatch):
    fake_etccdi.install(monkeypatch)
    from xclim_b200 import Field, indices
    tx = make_field(np.zeros((365, 2), np.float32), "2001-01-01", calendar="noleap", units="K")
    per = _per_field(np.zeros((365, 2)), "K")
    for fn in (indices.warm_spell_duration_index, indices.cold_spell_duration_index,
               indices.fraction_over_precip_thresh):
        with pytest.raises(NotImplementedError, match="bootstrap"):
            fn(tx, per, bootstrap=True)
    with pytest.raises(ValueError, match="not permitted"):
        indices.warm_spell_duration_index(tx, per, op="<")
    with pytest.raises(ValueError, match="not permitted"):
        indices.cold_spell_duration_index(tx, per, op=">=")
    with pytest.raises(ValueError, match="not permitted"):
        indices.fraction_over_precip_thresh(tx, per, op="<")
    no_doy = Field(np.zeros((2, 365)), ("d0", "x"), None, {}, {"units": "K"})
    with pytest.raises(AttributeError, match="dayofyear"):
        indices.warm_spell_duration_index(tx, no_doy)
    with pytest.raises(AttributeError, match="dayofyear"):
        indices.cold_and_dry_days(tx, tx, no_doy, per)
    c = make_field(np.zeros((365, 2), np.float32), "2001-01-01", calendar="noleap", units="degC")
    for fn in (indices.daily_temperature_range, indices.daily_temperature_range_variability):
        with pytest.raises(NotImplementedError, match="same units"):
            fn(c, tx)
    with pytest.raises(NotImplementedError):
        indices.daily_temperature_range(tx, tx, op=np.mean)


def test_indicator_and_dataarray_boundary(monkeypatch):
    """atmos.<name> is built on first use (MissingAny); a mini-xarray DataArray comes back as one."""
    fake_etccdi.install(monkeypatch)
    from xclim_b200 import atmos
    lo = np.full((365, 2), 270.0, np.float32)
    hi = lo + 10
    hi[40, 0] = np.nan
    a = make_field(lo, "2001-01-01", calendar="noleap", units="K")
    b = make_field(hi, "2001-01-01", calendar="noleap", units="K")
    out = atmos.daily_temperature_range(a, b, freq="MS").values
    assert np.isnan(out[1, 0]) and out[1, 1] == 10 and out[0, 0] == 10


# ------------------------------------------------------------------ the C entry points check their arguments
@pytest.fixture(scope="module")
def lib():
    import os

    from xclim_b200 import _build, _lib
    if not os.path.exists(_build.LIB_PATH):
        _build.build()
    return _lib.load()


def test_entry_points_validate_on_the_host(lib):
    INVALID = -1
    buf = (C.c_float * 64)()
    ibuf = (C.c_int32 * 16)(0, 4)
    dbuf = (C.c_double * 64)()
    sbuf = (C.c_int16 * 16)(1, 2, 3, 4)
    p, ip, dp, sp = (C.cast(b, C.c_void_p) for b in (buf, ibuf, dbuf, sbuf))
    # run statistic against a table
    args = [p, 4, 4, 4, ip, 1, sp, dp, 4]
    assert lib.xc_doy_runstat_f32(None, *args[1:], 0, 2, 1, 1, p, None, None) == INVALID
    assert b"null pointer" in lib.xc_last_error()
    assert lib.xc_doy_runstat_f32(*args[:6], None, dp, 4, 0, 2, 1, 1, p, None, None) == INVALID
    assert lib.xc_doy_runstat_f32(p, 4, 4, 2, ip, 1, sp, dp, 4, 0, 2, 1, 1, p, None, None) == INVALID
    assert b"shape" in lib.xc_last_error()
    assert lib.xc_doy_runstat_f32(*args, 4, 2, 1, 1, p, None, None) == INVALID          # == is not a spell test
    assert b"not permitted" in lib.xc_last_error()
    assert lib.xc_doy_runstat_f32(*args, 0, 9, 1, 1, p, None, None) == INVALID
    assert b"reducer" in lib.xc_last_error()
    assert lib.xc_doy_runstat_f32(*args, 0, 2, 0, 1, p, None, None) == INVALID
    assert b"window" in lib.xc_last_error()
    assert lib.xc_doy_runstat_f32(*args[:8], 0, 0, 2, 1, 1, p, None, None) == INVALID
    assert lib.xc_doy_runstat_f32(*args[:5], 0, *args[6:], 0, 2, 1, 1, p, None, None) == INVALID
    # the two sums
    args = [p, 4, 4, 4, ip, 1, sp, dp]
    assert lib.xc_period_sums_thr_f32(*args, 4, 0, 1.0, p, None, None) == INVALID
    assert b"null pointer" in lib.xc_last_error()
    assert lib.xc_period_sums_thr_f32(*args, 2, 0, 1.0, p, p, None) == INVALID
    assert b"stride" in lib.xc_last_error()
    assert lib.xc_period_sums_thr_f32(*args, 4, 1, 1.0, p, p, None) == INVALID
    assert b"not permitted" in lib.xc_last_error()
    assert lib.xc_period_sums_thr_f32(p, 4, 4, 4, ip, 70000, sp, dp, 4, 0, 1.0, p, p, None) == INVALID
    # the compound count
    args = [p, p, 4, 4, 4, ip, 1, sp, dp, dp, 4]
    assert lib.xc_doy_count2_f32(*args[:7], None, dp, dp, 4, 0, 1, p, None) == INVALID
    assert b"null pointer" in lib.xc_last_error()
    assert lib.xc_doy_count2_f32(*args, 0, 5, p, None) == INVALID
    assert b"not permitted" in lib.xc_last_error()
    assert lib.xc_doy_count2_f32(*args[:10], 0, 0, 1, p, None) == INVALID
    assert b"shape" in lib.xc_last_error()
    # the daily range
    args = [p, p, 4, 4, 4, ip, 1]
    assert lib.xc_period_range_stat_f32(*args, 9, 0, p, None) == INVALID
    assert b"reduction" in lib.xc_last_error()
    assert lib.xc_period_range_stat_f32(*args, 3, 1, p, None) == INVALID
    assert b"variability" in lib.xc_last_error()
    assert lib.xc_period_range_stat_f32(p, None, 4, 4, 4, ip, 1, 1, 0, p, None) == INVALID
    assert lib.xc_period_range_stat_f32(p, p, 0, 4, 4, ip, 1, 1, 0, p, None) == INVALID
