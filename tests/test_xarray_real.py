"""The same boundary with the REAL xarray (and, when importable, the real xclim registry).  Skipped where
xarray is not installed (this image); engages by itself on a box that has it."""
import numpy as np
import pytest

xr = pytest.importorskip("xarray")

from oracle import xclim_oracle as O   # noqa: E402

pytestmark = pytest.mark.gpu


def _da(values, units, calendar="noleap"):
    T = values.shape[0]
    time = xr.date_range("2001-01-01", periods=T, freq="D", calendar=calendar, use_cftime=True)
    return xr.DataArray(values, dims=("time", "lat", "lon"),
                        coords={"time": time, "lat": np.arange(values.shape[1]) * 0.25,
                                "lon": np.arange(values.shape[2]) * 0.25}, attrs={"units": units})


def _data():
    rng = np.random.default_rng(92)
    T, shape = 365 * 3, (3, 5)
    t = np.arange(T)
    tas = (285 + 10 * np.sin(2 * np.pi * (t % 365 - 110) / 365)[:, None, None]
           + 3 * rng.standard_normal((T,) + shape)).astype(np.float32)
    pr = rng.gamma(0.4, 6.0, size=(T,) + shape).astype(np.float32)
    pr[rng.random(pr.shape) < 0.5] = 0
    return tas, pr


def test_dataarrays_in_dataarrays_out(cuda):
    from xclim_b200 import TimeAxis, calendar as xcal, indices
    tas, pr = _data()
    ta = TimeAxis.daily("2001-01-01", tas.shape[0], "noleap")
    poff = ta.period_offsets("YS")
    cdd = indices.maximum_consecutive_dry_days(_da(pr, "mm/d"), thresh="1 mm/day", freq="YS")
    assert isinstance(cdd, xr.DataArray) and cdd.dims == ("time", "lat", "lon") and cdd.sizes["time"] == 3
    np.testing.assert_array_equal(cdd.values, O.maximum_consecutive_dry_days(pr, 1.0, poff))
    per = xcal.percentile_doy(_da(tas, "K"), window=5, per=90.0)
    assert per.dims == ("lat", "lon", "dayofyear", "percentiles")
    tx = indices.tx90p(_da(tas, "K"), per.sel(percentiles=90.0), freq="YS")
    tab = O.percentile_doy(tas, ta.year, ta.doy, 5, 90.0)[:, 0]
    np.testing.assert_array_equal(tx.values, O.doy_threshold_count(tas, tab, ta.doy, poff, ">"))


def test_registered_under_the_xclim_indicator_registry(cuda):
    """INTEGRATION.md route (a): bind the xclim_b200 index as ``compute`` of a stock indicator and compare with
    stock xclim on the same input (engages only where xclim imports)."""
    xclim = pytest.importorskip("xclim")
    from xclim.core.indicator import Indicator
    from xclim_b200 import indices
    _, pr = _data()
    da = _da(pr, "mm/d")
    da.attrs.update(standard_name="precipitation_flux", cell_methods="time: mean")
    ref = xclim.atmos.maximum_consecutive_dry_days(da, thresh="1 mm/day", freq="YS")
    ind = Indicator.from_dict({"base": "cdd", "compute": indices.maximum_consecutive_dry_days},
                              identifier="cdd_b200", module="b200")
    got = ind(da, thresh="1 mm/day", freq="YS")
    np.testing.assert_array_equal(got.values, ref.values)
