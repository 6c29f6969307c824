"""Potential evapotranspiration and the water budget against the REAL xclim (xarray, pint, cftime) at 1e-6 relative.
Skipped where xclim is not installed; engages by itself on a machine that has it.  This checks what the other tests
cannot: pint's unit factors (cal, MJ, W m-2, mm/d, its ``month``) and xarray's ``dt.decimal_year``."""
import numpy as np
import pytest

xr = pytest.importorskip("xarray")
xci = pytest.importorskip("xclim.indices")

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore::RuntimeWarning")]

UNITS = {"tasmin": "K", "tasmax": "K", "tas": "K", "hurs": "%", "rsds": "W m-2", "rsus": "W m-2", "rlds": "W m-2",
         "rlus": "W m-2", "sfcWind": "m s-1", "pr": "kg m-2 s-1"}


def _data(calendar):
    rng = np.random.default_rng(5)
    T, nl, nx = 2 * 365, 4, 3
    time = xr.date_range("2001-01-01", periods=T, freq="D", calendar=calendar, use_cftime=True)
    lat = xr.DataArray(np.array([-50.0, 0.0, 45.0, 70.0]), dims="lat",
                       attrs={"standard_name": "latitude", "units": "degrees_north"})
    season = 10 * np.sin(2 * np.pi * (np.arange(T) % 365 - 110) / 365)[:, None, None]
    tn = 275 + season + 3 * rng.standard_normal((T, nl, nx))
    vals = {"tasmin": tn, "tasmax": tn + rng.uniform(2, 12, (T, nl, nx)), "hurs": rng.uniform(20, 100, (T, nl, nx)),
            "rsds": rng.uniform(20, 350, (T, nl, nx)), "rsus": rng.uniform(5, 60, (T, nl, nx)),
            "rlds": rng.uniform(220, 380, (T, nl, nx)), "rlus": rng.uniform(240, 420, (T, nl, nx)),
            "sfcWind": rng.uniform(0.5, 12, (T, nl, nx)), "pr": rng.gamma(0.6, 4e-5, (T, nl, nx))}
    vals["tas"] = (vals["tasmin"] + vals["tasmax"]) / 2
    coords = {"time": time, "lat": lat, "lon": np.arange(nx) * 1.0}
    return {k: xr.DataArray(v.astype(np.float32), dims=("time", "lat", "lon"), coords=coords, name=k,
                            attrs={"units": UNITS[k]}) for k, v in vals.items()}


def _close(got, ref):
    got, ref = np.asarray(got.values, np.float64), np.asarray(ref.values, np.float64)
    assert got.shape == ref.shape
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    ok = ~np.isnan(ref)
    np.testing.assert_allclose(got[ok], ref[ok], rtol=1e-6, atol=1e-6 * np.abs(ref[ok]).max())


@pytest.mark.parametrize("calendar", ["noleap", "standard", "360_day"])
@pytest.mark.parametrize("method,names", [
    ("BR65", ("tasmin", "tasmax")), ("HG85", ("tasmin", "tasmax", "tas")), ("MB05", ("tas",)),
    ("FAO_PM98", ("tasmin", "tasmax", "hurs", "rsds", "rsus", "rlds", "rlus", "sfcWind")), ("TW48", ("tas",)),
    ("DA02", ("tasmin", "tasmax", "pr"))])
def test_potential_evapotranspiration_matches_xclim(calendar, method, names):
    from xclim_b200 import indices
    d = _data(calendar)
    kw = {k: d[k] for k in names}
    ref = xci.potential_evapotranspiration(method=method, **kw)
    got = indices.potential_evapotranspiration(method=method, **kw)
    assert isinstance(got, xr.DataArray) and got.dims == ref.dims
    _close(got, ref)


@pytest.mark.parametrize("method,names", [("BR65", ("tasmin", "tasmax")), ("HG85", ("tasmin", "tasmax")),
                                          ("TW48", ("tas",))])
def test_water_budget_matches_xclim(method, names):
    from xclim_b200 import indices
    d = _data("noleap")
    kw = {k: d[k] for k in names}
    _close(indices.water_budget(d["pr"], method=method, **kw), xci.water_budget(d["pr"], method=method, **kw))
    pet = xci.potential_evapotranspiration(tasmin=d["tasmin"], tasmax=d["tasmax"], method="BR65")
    _close(indices.water_budget(d["pr"], evspsblpot=pet.astype(np.float32).assign_attrs(units="kg m-2 s-1")),
           xci.water_budget(d["pr"], evspsblpot=pet.astype(np.float32).assign_attrs(units="kg m-2 s-1")))
