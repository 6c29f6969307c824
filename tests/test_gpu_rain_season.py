"""GPU parity of the rain-season kernel (xc_rain_season_f32): bit for bit against the host build of its scan and the
oracle on the seeded cases, around whole CTAs (1 to 4100 cells), on column views (ldx > C), for 1 to 40 periods on
every calendar and annual anchor; the known answers through indices.rain_season, the indicator with NaN days, and the
streamed host path."""
import numpy as np
import pytest

import rain_season_cases as cases
from oracle import rain_season_oracle as R
from test_rain_season_cpu import KNOWN, KNOWN_KW, host_build, known_series
from xb_helpers import make_field
from xclim_b200 import _lib
from xclim_b200.timeaxis import TimeAxis

pytestmark = pytest.mark.gpu


def _kernel(x_dev, ta, freq, scale, params):
    from xclim_b200 import device
    from xclim_b200.indices import _rain_season_mask
    p = {**R.DEFAULTS, **params}
    poff = ta.period_offsets(freq)
    mask = _rain_season_mask(ta, poff, p["date_min_start"], p["date_max_start"], p["date_min_end"], p["date_max_end"])
    s, e = device.rain_season(x_dev, poff, mask, scale, p["thresh_wet_start"], p["window_wet_start"],
                              p["window_not_dry_start"], p["thresh_dry_start"], p["window_dry_start"],
                              _lib.RS_METHODS[p["method_dry_start"]], p["thresh_dry_end"], p["window_dry_end"],
                              _lib.RS_METHODS[p["method_dry_end"]])
    s, e = s.cpu().numpy(), e.cpu().numpy()
    return np.where(s < 0, np.nan, s), np.where(e < 0, np.nan, e)


def _views(x):
    """Contiguous, and a column slice of a wider buffer (ldx > C)."""
    import torch
    T, C = x.shape
    wide = torch.full((T, C + 37), float("nan"), device="cuda")
    wide[:, 5:C + 5] = torch.from_numpy(x).cuda()
    return [("contiguous", torch.from_numpy(x).cuda()), ("ldx", wide[:, 5:C + 5])]


@pytest.mark.parametrize("method", ["per_day", "total"])
def test_kernel_matches_host_build_and_oracle(cuda, method):
    n = 0
    for x, ta, freq, scale, params in cases.cases(21 if method == "per_day" else 22, method, 48):
        try:
            o = R.rain_season(x, ta, freq, scale, **params)
        except ValueError:
            continue
        hs, he = host_build(x, ta, freq, scale, params)
        np.testing.assert_array_equal(hs, o["start_idx"], err_msg=str(params))
        np.testing.assert_array_equal(he, o["end_idx"], err_msg=str(params))
        for name, v in _views(x):
            s, e = _kernel(v, ta, freq, scale, params)
            np.testing.assert_array_equal(s, hs, err_msg=f"{name} {params}")
            np.testing.assert_array_equal(e, he, err_msg=f"{name} {params}")
        n += hs.size
    assert n >= 10000


@pytest.mark.parametrize("calendar", ["noleap", "360_day", "all_leap", "standard"])
@pytest.mark.parametrize("freq", ["YS-JAN", "YS-JUL"])
@pytest.mark.parametrize("C,years", [(1, 1), (127, 3), (128, 40), (129, 7), (4100, 12)])
def test_grid_edges(cuda, calendar, freq, C, years):
    rng = np.random.default_rng(C * 7 + years)
    start = "1990-01-01" if freq == "YS-JAN" else "1990-07-01"
    ta = TimeAxis.daily(start, years * 366, calendar)
    ta = ta.isel(slice(0, int(ta.period_offsets(freq)[years])))
    params = dict(R.DEFAULTS, thresh_wet_start=20.0, window_not_dry_start=20, date_min_start="03-01",
                  date_min_end="07-01", method_dry_end=("per_day", "total")[C % 2], thresh_dry_end=0.5,
                  window_dry_end=10)
    for k in ("thresh_wet_start", "thresh_dry_start", "thresh_dry_end"):
        params[k] = float(params[k])
    x = cases.series(rng, len(ta), C, params, 1.0)
    poff = ta.period_offsets(freq)
    assert len(poff) - 1 == years
    hs, he = host_build(x, ta, freq, 1.0, params)
    for name, v in _views(x):
        s, e = _kernel(v, ta, freq, 1.0, params)
        np.testing.assert_array_equal(s, hs, err_msg=name)
        np.testing.assert_array_equal(e, he, err_msg=name)
    cols = sorted({0, C // 2, C - 1, min(C - 1, 127), min(C - 1, 128)})
    o = R.rain_season(x[:, cols], ta, freq, 1.0, **params)
    np.testing.assert_array_equal(hs[:, cols], o["start_idx"])
    np.testing.assert_array_equal(he[:, cols], o["end_idx"])
    assert np.isfinite(hs).mean() > 0.2


@pytest.mark.parametrize("method_dry_start", ["per_day", "total"])
@pytest.mark.parametrize("result_type", list(KNOWN))
def test_known_answers(cuda, result_type, method_dry_start):
    from xclim_b200 import indices
    pr = make_field(known_series(result_type)[:, None], "2000-01-01", "standard", units="mm/d")
    out = indices.rain_season(pr, method_dry_start=method_dry_start, **KNOWN_KW)
    np.testing.assert_array_equal([np.asarray(o.values)[0, 0] for o in out], KNOWN[result_type])


def test_indicator_with_nan_days(cuda):
    """atmos.rain_season: the oracle's three outputs, NaN in every period where a day is missing (MissingAny)."""
    from xclim_b200 import atmos
    rng = np.random.default_rng(8)
    params = dict(date_min_start="03-01", date_min_end="07-01")
    x = cases.series(rng, 365 * 3, 300, dict(R.DEFAULTS), 86400.0)
    x[rng.random(x.shape) < 0.0005] = np.nan
    ta = TimeAxis.daily("2001-01-01", 365 * 3, "noleap")
    out = atmos.rain_season(make_field(x, "2001-01-01", "noleap", units="kg m-2 s-1"), **params)
    o = R.rain_season(x, ta, "YS-JAN", 86400.0, **params)
    poff = ta.period_offsets("YS-JAN")
    miss = np.stack([np.isnan(x[a:b]).any(0) for a, b in zip(poff[:-1], poff[1:])])
    assert miss.any() and (~miss).any()
    for got, key in zip(out, ("start", "end", "length")):
        np.testing.assert_array_equal(np.asarray(got.values), np.where(miss, np.nan, o[key]), err_msg=key)


def test_streamed_host_input_matches_device_resident(cuda):
    import torch

    import xclim_b200
    from xclim_b200 import Field, indices
    rng = np.random.default_rng(12)
    ta = TimeAxis.daily("2001-01-01", 365 * 2, "noleap")
    T, nl, nx = len(ta), 9, 40
    x = cases.series(rng, T, nl * nx, dict(R.DEFAULTS), 1.0).reshape(T, nl, nx)
    host = Field(x, ("time", "lat", "lon"), ta, {}, {"units": "mm/d"})
    dev = Field(torch.from_numpy(x).cuda(), ("time", "lat", "lon"), ta, {}, {"units": "mm/d"})
    with xclim_b200.set_options(stream_min_bytes=1, stream_slab_bytes=T * nx * 4 * 2):
        streamed = indices.rain_season(host, date_min_start="03-01")
    with xclim_b200.set_options(device_outputs=True):
        resident = indices.rain_season(dev, date_min_start="03-01")
    for s, r in zip(streamed, resident):
        np.testing.assert_array_equal(np.asarray(s.values), r.values.cpu().numpy())
        assert s.dims == ("time", "lat", "lon")
    assert np.isfinite(np.asarray(streamed[0].values)).any()
