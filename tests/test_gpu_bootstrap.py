"""GPU parity: percentile bootstrap (core/bootstrapping.py) vs the literal CPU restatement."""
import numpy as np
import pytest

from oracle import xclim_oracle as O
from xb_helpers import make_field, plant_infinite_samples

pytestmark = pytest.mark.gpu


def _tas(rng, T, shape, nan_frac=0.0):
    t = np.arange(T)
    x = 288 + 12 * np.sin(2 * np.pi * (t % 365 - 110) / 365)[(slice(None),) + (None,) * len(shape)]
    x = (x + 3 * rng.standard_normal((T,) + shape)).astype(np.float32)
    if nan_frac:
        x[rng.random(x.shape) < nan_frac] = np.nan
    return x


@pytest.mark.parametrize("nbase,nyears,per,op,freq", [
    (5, 8, 90.0, ">", "YS"),
    (6, 7, 10.0, "<", "YS"),
    (4, 6, 90.0, ">=", "MS"),
    (15, 17, 90.0, ">", "YS"),
])
def test_bootstrap_matches_literal_restatement(cuda, nbase, nyears, per, op, freq):
    from xclim_b200 import calendar as xcal, indices
    rng = np.random.default_rng(31)
    shape = (3, 4) if nbase < 10 else (2, 2)
    x = _tas(rng, 365 * nyears, shape, nan_frac=0.004)
    x[:, 0, 0] = np.round(x[:, 0, 0])          # many exact ties
    da = make_field(x, "1981-01-01", calendar="noleap", units="K")
    base = da.isel_time(da.time.sel_years(1982, 1982 + nbase - 1))  # base does not start at the series start
    pdoy = xcal.select_percentile(xcal.percentile_doy(base, window=5, per=per), per)
    fn = indices.tx90p if op in (">", ">=") else indices.tx10p
    got = fn(da, pdoy, freq=freq, bootstrap=True, op=op)
    exp = O.bootstrap_doy_count(x, da.time.year, da.time.doy, da.time.period_offsets(freq),
                                (1982, 1982 + nbase - 1), window=5, per=per, op=op)
    assert got.values.dtype == np.float64 and got.attrs["units"] == "d"
    np.testing.assert_array_equal(got.values, exp)   # integer sums / (N-1): bit-exact
    # the property the reference pins (tests/test_bootstrapping.py:65-71): out-of-base years equal the plain index
    plain = fn(da, pdoy, freq=freq, bootstrap=False, op=op).values.astype(np.float64)
    yrs = np.array([int(s[:4]) for s in da.time.period_labels(freq)])
    outside = (yrs < 1982) | (yrs > 1982 + nbase - 1)
    np.testing.assert_array_equal(got.values[outside], plain[outside])
    assert (got.values[~outside] != plain[~outside]).any()


def test_bootstrap_error_behaviour(cuda):
    """core/bootstrapping.py:131-168."""
    from xclim_b200 import calendar as xcal, indices, Field
    rng = np.random.default_rng(32)
    x = _tas(rng, 365 * 4, (2, 2))
    da = make_field(x, "1981-01-01", calendar="noleap", units="K")
    p_all = xcal.select_percentile(xcal.percentile_doy(da, per=90.0), 90.0)
    with pytest.raises(KeyError, match="all years are overlapping"):
        indices.tx90p(da, p_all, bootstrap=True)
    other = make_field(x, "1991-01-01", calendar="noleap", units="K")
    with pytest.raises(KeyError, match="no year overlap"):
        indices.tx90p(other, p_all, bootstrap=True)
    nohist = Field(p_all.values, p_all.dims, None, dict(p_all.coords), {"units": "K"})
    with pytest.raises(KeyError, match="percentile_doy"):
        indices.tx90p(da, nohist, bootstrap=True)


@pytest.mark.parametrize("per,op,freq", [(90.0, ">", "YS"), (10.0, "<", "MS")])
def test_bootstrap_standard_calendar_365_366_blocks(cuda, per, op, freq):
    """Year blocks of unequal length (core/bootstrapping.py:266-269): a 365-day block replaced by a leap
    year loses its Feb 29, a 366-day block replaced by a common year gets NaN on Feb 29; tables go
    through the 366-doy machinery + interpolation (core/calendar.py:484-485)."""
    from xclim_b200 import calendar as xcal, indices
    rng = np.random.default_rng(33)
    ta_len = 366 + 365 * 3 + 366 + 365 * 2          # 2000 .. 2006 (leap: 2000, 2004)
    x = _tas(rng, ta_len, (2, 3), nan_frac=0.004)
    x[:, 0, 0] = np.round(x[:, 0, 0])
    da = make_field(x, "2000-01-01", calendar="standard", units="K")
    assert len(da.time) == ta_len
    y0, y1 = 2001, 2005                              # base holds one leap year and four common years
    base = da.isel_time(da.time.sel_years(y0, y1))
    pdoy = xcal.select_percentile(xcal.percentile_doy(base, window=5, per=per), per)
    fn = indices.tx90p if op in (">", ">=") else indices.tx10p
    got = fn(da, pdoy, freq=freq, bootstrap=True, op=op)
    exp = O.bootstrap_doy_count(x, da.time.year, da.time.doy, da.time.period_offsets(freq), (y0, y1), window=5,
                                per=per, op=op, cal_max_doy=366)
    np.testing.assert_array_equal(got.values, exp)
    plain = fn(da, pdoy, freq=freq, bootstrap=False, op=op).values.astype(np.float64)
    yrs = np.array([int(s[:4]) for s in da.time.period_labels(freq)])
    outside = (yrs < y0) | (yrs > y1)
    np.testing.assert_array_equal(got.values[outside], plain[outside])


def _raw_doy_table(x, year, doy, window, pers):
    """(n_per, 366, C) day-of-year quantiles of O.percentile_doy before its 365 -> 366 re-interpolation"""
    rr = O.rolling_construct_center(x, window)
    ny = int(year.max()) + 1
    rrr = np.full((366, ny * window) + x.shape[1:], np.nan, dtype=rr.dtype)
    for t in range(x.shape[0]):
        rrr[doy[t] - 1, year[t] * window:(year[t] + 1) * window] = rr[t]
    q = np.stack([O.nan_quantile(rrr[d], np.asarray(pers) / 100.0, 1 / 3, 1 / 3) for d in range(366)])
    return np.moveaxis(q, 1, 0)


def test_percentile_vrow_identity_and_replacement(cuda):
    """xc_percentile_doy_vrow_f32: the identity map reproduces the plain table bit for bit, and a block
    replacement equals the table of a physically modified copy of the series."""
    from xclim_b200 import device as dv
    import torch
    rng = np.random.default_rng(34)
    T = 366 + 365 * 3 + 366
    x = _tas(rng, T, (17,), nan_frac=0.01)
    plant_infinite_samples(x, [0.9, 0.1], range(7, 17), seed=34)
    da = make_field(x, "2000-01-01", calendar="standard", units="K")
    ta = da.time
    years = np.unique(ta.year)
    yidx = np.searchsorted(years, ta.year).astype(np.int16)
    xd = torch.from_numpy(x).cuda()
    plain = dv.percentile_doy(xd, ta.doy, yidx, 366, len(years), 5, [90.0, 10.0], 1 / 3, 1 / 3)
    np.testing.assert_array_equal(plain.cpu().numpy(), _raw_doy_table(x, yidx, ta.doy, 5, [90.0, 10.0]))
    ident = dv.percentile_doy(xd, ta.doy, yidx, 366, len(years), 5, [90.0, 10.0], 1 / 3, 1 / 3,
                              vrow=np.arange(T, dtype=np.int32))
    assert torch.equal(plain.view(torch.int64), ident.view(torch.int64))
    # year 2001 (365 days, rows 366..730) <- year 2004 (366 days) without its Feb 29
    a, src0 = 366, 366 + 365 * 3
    rows = np.delete(src0 + np.arange(366), 59)
    vrow = np.arange(T, dtype=np.int32)
    vrow[a:a + 365] = rows
    z = x.copy()
    z[a:a + 365] = x[rows]
    got = dv.percentile_doy(xd, ta.doy, yidx, 366, len(years), 5, [90.0], 1 / 3, 1 / 3, vrow=vrow)
    ref = dv.percentile_doy(torch.from_numpy(z).cuda(), ta.doy, yidx, 366, len(years), 5, [90.0], 1 / 3, 1 / 3)
    assert torch.equal(got.view(torch.int64), ref.view(torch.int64))
    np.testing.assert_array_equal(got.cpu().numpy(), _raw_doy_table(z, yidx, ta.doy, 5, [90.0]))
    # year 2000 (366 days, rows 0..365) <- year 2002 with NaN on Feb 29
    src0 = 366 + 365
    rows = np.insert(src0 + np.arange(365), 59, -1)
    vrow = np.arange(T, dtype=np.int32)
    vrow[0:366] = rows
    z = x.copy()
    z[0:366] = np.where((rows >= 0)[:, None], x[np.maximum(rows, 0)], np.nan)
    got = dv.percentile_doy(xd, ta.doy, yidx, 366, len(years), 5, [90.0], 1 / 3, 1 / 3, vrow=vrow)
    ref = dv.percentile_doy(torch.from_numpy(z).cuda(), ta.doy, yidx, 366, len(years), 5, [90.0], 1 / 3, 1 / 3)
    assert torch.equal(got.view(torch.int64), ref.view(torch.int64))
