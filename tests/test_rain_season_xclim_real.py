"""The rain season against the REAL xclim (xarray, pint, cftime) at exact equality.  Skipped where xclim is not
installed; engages by itself on a machine that has it.  The series hold quarter-mm amounts in mm/d, so every window
sum is exact in float32 as in float64 and the outputs must agree exactly."""
import numpy as np
import pytest

import rain_season_cases as cases

xr = pytest.importorskip("xarray")
xci = pytest.importorskip("xclim.indices")

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("calendar", ["noleap", "360_day", "standard"])
@pytest.mark.parametrize("method", ["per_day", "total"])
def test_rain_season_matches_xclim(cuda, calendar, method):
    from xclim_b200 import indices
    from oracle import rain_season_oracle as R
    params = dict(R.DEFAULTS, method_dry_start=method, method_dry_end=method, date_min_start="03-01")
    T = 3 * 360 if calendar == "360_day" else 3 * 365
    x = cases.series(np.random.default_rng(4), T, 64, params, 1.0)
    x[~np.isfinite(x)] = 0                      # finite, quarter-mm amounts: exact window sums
    x = np.abs(np.round(x * 4) / 4).astype(np.float32)
    time = xr.date_range("2001-01-01", periods=T, freq="D", calendar=calendar, use_cftime=True)
    pr = xr.DataArray(x, dims=("time", "cell"), coords={"time": time}, name="pr", attrs={"units": "mm/d"})
    kw = {k: (f"{v} mm" if k.startswith("thresh") else v) for k, v in params.items()}
    ref = xci.rain_season(pr, **kw)
    got = indices.rain_season(pr, **kw)
    for g, r in zip(got, ref):
        np.testing.assert_array_equal(np.asarray(g.values, np.float64), np.asarray(r.values, np.float64))
