"""The standardized-index host layer (xclim_b200/stats.py, the SPI / SPEI entry points) on the CPU: the device
functions are replaced by stand-ins (fake_device for the staging and monthly means, oracle/stdindex_oracle.py
for the rolling mean, the host build of stdindex_core.cuh for the fit and the transform), so the preprocessing,
grouping, calibration slices, indexers, params round trip, containers, attrs and errors are exercised here;
the kernels themselves are checked by test_gpu_stdindex.py.  Also the argument checks of the new C entry
points (no device work)."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest
import scipy.stats as st
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import fake_device  # noqa: E402
import mini_xarray as mx  # noqa: E402
import stdindex_host_build as H  # noqa: E402
from oracle import stdindex_oracle as O  # noqa: E402

pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")
DIST_NAME = {0: "gamma", 1: "fisk", 2: "lognorm"}
METHOD_NAME = {0: "APP", 1: "ML"}


def fake_rolling_mean(x2d, window):
    return torch.from_numpy(O.rolling_mean(x2d.numpy(), int(window)))


def fake_si_fit(x2d, group_offsets, steps, dist_code, method_code, zero_inflated, floc):
    y = np.ascontiguousarray(x2d.numpy(), dtype=np.float32)
    T, Cn = y.shape
    goff = np.ascontiguousarray(group_offsets, dtype=np.int32)
    st_ = np.ascontiguousarray(steps if len(steps) else np.zeros(1), dtype=np.int32)
    G = goff.size - 1
    params = np.empty((G, 3, Cn))
    nz = np.zeros((G, Cn), np.int32)
    nn = np.zeros((G, Cn), np.int32)
    ws = np.empty(max(1, int(np.diff(goff).max())) * Cn, np.float32)
    p_ = H._p
    status = H.load().si_host_fit(p_(y), Cn, Cn, p_(goff), p_(st_), G, dist_code, method_code, int(zero_inflated),
                                  float(floc), p_(params), p_(nz), p_(nn), p_(ws))
    zi = bool(zero_inflated)
    return (torch.from_numpy(params), torch.from_numpy(nz) if zi else None, torch.from_numpy(nn) if zi else None,
            int(status))


def fake_si_apply(x2d, group_of_step, params, n_zeros, n_notnull, dist_code, interp=1.0, alpha=0.0, beta=1.0):
    out = H.apply(x2d.numpy(), np.asarray(group_of_step), params.numpy(), DIST_NAME[dist_code],
                  None if n_zeros is None else n_zeros.numpy(), None if n_notnull is None else n_notnull.numpy(),
                  interp, alpha, beta)
    return torch.from_numpy(out)


@pytest.fixture
def host(monkeypatch):
    from xclim_b200 import device
    fake_device.install(monkeypatch)
    monkeypatch.setattr(device, "rolling_mean", fake_rolling_mean)
    monkeypatch.setattr(device, "si_fit", fake_si_fit)
    monkeypatch.setattr(device, "si_apply", fake_si_apply)


def _field(values, start="1981-01-01", calendar="noleap"):
    from xclim_b200.field import Field
    from xclim_b200.timeaxis import TimeAxis
    ta = TimeAxis.daily(start, values.shape[0], calendar)
    return Field(values, ("time", "lat", "lon"), ta, {}, {"units": "mm/d"})


def _pr(days, seed=0, shape=(2, 3)):
    rng = np.random.default_rng(seed)
    pr = rng.gamma(0.5, 6.0, (days,) + shape).astype(np.float32)
    pr[rng.random(pr.shape) < 0.4] = 0.0
    pr[3:40, 0, 0] = np.nan
    return pr


def _expected(pr, ta, freq, window, dist, method, zi, cal=(None, None), keep=None, floc=0.0):
    """The pipeline restated: monthly NaN-skipping means (fake_device's), the oracle's rolled series, groups,
    the oracle fit (kernel log rule) and transform."""
    from xclim_b200 import stats
    T = pr.shape[0]
    x = pr.reshape(T, -1)
    if freq == "MS":
        poff = ta.period_offsets("MS")
        y = fake_device.period_reduce(torch.from_numpy(x), poff, 1)[0].numpy()
        gid = ta.month[poff[:-1]] - 1
        G = 12
        year, month, day = ta.year[poff[:-1]], ta.month[poff[:-1]], np.ones(poff.size - 1, np.int32)
    else:
        y, gid, G = x, ta.doy - 1, ta.max_doy
        year, month, day = ta.year, ta.month, ta.day
    y = O.rolling_mean(y, window)
    keep = np.ones(len(gid), bool) if keep is None else keep
    s = stats._Series(None, year, month, day, None, gid, None, G, ta.calendar, None)
    cs = stats._cal_slice(s, *cal)
    gfit = np.where(keep, gid, -1)
    if method == "ML":   # the ML shape is a root, equal to the oracle's only within brentq's tolerance
        p, nz, nn, _ = H.fit(y, gfit, G, dist, method, zi, floc, cs)
    else:
        p, nz, nn = O.fit_groups(y, gfit, G, cs, dist, method, zi, floc, numpy_logs=False)
    present = np.unique(gid[cs])
    gos = np.where(keep & np.isin(gid, present), gid, -1)
    return O.transform(y, gos, p, dist, nz if zi else None, nn if zi else None), p, present


def _close(out, exp):
    out = np.asarray(out).reshape(exp.shape)
    np.testing.assert_array_equal(np.isnan(out), np.isnan(exp))
    ok = ~np.isnan(exp)
    assert np.all(np.abs(out - exp)[ok] * st.norm.pdf(exp[ok]) <= 1e-13)


@pytest.mark.parametrize("freq,window", [("MS", 1), ("MS", 3), ("MS", 12), ("D", 1), ("D", 30), (None, 3)])
@pytest.mark.parametrize("dist,method", [("gamma", "ML"), ("fisk", "APP"), ("lognorm", "APP")])
def test_spi_against_restated_pipeline(host, freq, window, dist, method):
    from xclim_b200 import indices
    pr = _pr(365 * 6, seed=window)
    da = _field(pr)
    out = indices.standardized_precipitation_index(da, freq=freq, window=window, dist=dist, method=method,
                                                   fitkwargs={"floc": 0}, cal_start="1982", cal_end="1985-06")
    exp, _, _ = _expected(pr, da.time, freq, window, dist, method, True, cal=("1982", "1985-06"))
    _close(out.values, exp)
    assert out.dims == ("time", "lat", "lon")
    assert out.attrs["freq"] == (freq or "D") and out.attrs["window"] == window and out.attrs["units"] == ""
    assert out.attrs["calibration_period"] == (("1982-01-01", "1985-06-01") if freq == "MS" else
                                               ("1982-01-01", "1985-06-30"))


def test_spei_with_indexer_and_partial_calibration(host):
    from xclim_b200 import indices
    rng = np.random.default_rng(4)
    wb = rng.normal(1.0, 3.0, (365 * 5, 2, 2)).astype(np.float32)
    da = _field(wb)
    out = indices.standardized_precipitation_evapotranspiration_index(
        da, freq="MS", window=2, dist="fisk", method="APP", fitkwargs={"floc": -20.0}, cal_end="1984", month=[6, 7, 8])
    ta = da.time
    poff = ta.period_offsets("MS")
    keep = np.isin(ta.month[poff[:-1]], [6, 7, 8])
    exp, _, _ = _expected(wb, ta, "MS", 2, "fisk", "APP", False, cal=(None, "1984"), keep=keep, floc=-20.0)
    _close(out.values, exp)
    v = np.asarray(out.values)
    assert np.all(np.isnan(v[~keep])) and not np.all(np.isnan(v[keep]))


@pytest.mark.parametrize("freq,window", [("MS", 3), ("D", 1)])
def test_fit_params_container_and_round_trip(host, freq, window):
    from xclim_b200 import indices, stats
    pr = _pr(365 * 4, seed=9)
    da = _field(pr)
    params = stats.standardized_index_fit_params(da, freq=freq, window=window, dist="gamma", method="APP",
                                                 zero_inflated=True, fitkwargs={"floc": 0}, month=[1, 2, 3, 4, 5, 6])
    gdim = "month" if freq == "MS" else "dayofyear"
    assert params.dims == (gdim, "dparams", "lat", "lon")
    assert list(params.coords["dparams"]) == ["a", "loc", "scale"]
    assert np.asarray(params.values).dtype == np.float64
    np.testing.assert_array_equal(params.coords[gdim], np.arange(1, 13 if freq == "MS" else 366))
    z, n = params.coords["number_of_zeros"], params.coords["number_of_notnull"]
    assert z.dtype == np.int64 and n.dtype == np.int64 and z.shape == params.shape[:1] + params.shape[2:]
    np.testing.assert_array_equal(params.coords["prob_of_zero"], z / n)
    assert params.attrs == {"calibration_period": ("1981-01-01", params.attrs["calibration_period"][1]),
                            "freq": freq, "window": window, "scipy_dist": "gamma", "method": "APP",
                            "group": f"time.{gdim}", "units": "", "time_indexer": json.dumps({"month": [1, 2, 3, 4, 5, 6]})}
    # months outside the indexer have all-NaN parameters and no counted values
    mo = np.arange(12) + 1 if freq == "MS" else da.time.month[:365]
    assert np.all(np.isnan(np.asarray(params.values)[mo > 6])) and np.all(n[mo > 6] == 0)
    a = indices.standardized_precipitation_index(da, params=params)
    b = indices.standardized_precipitation_index(da, freq=freq, window=window, dist="gamma", method="APP",
                                                 fitkwargs={"floc": 0}, month=[1, 2, 3, 4, 5, 6])
    np.testing.assert_array_equal(np.asarray(a.values), np.asarray(b.values))


def test_xarray_boundary(host, monkeypatch):
    from xclim_b200 import indices, stats
    mx.install(monkeypatch)
    pr = _pr(365 * 3, seed=2)
    da = mx.daily(pr, "1981-01-01", units="mm/d")
    out = indices.standardized_precipitation_index(da, freq="MS", window=3, dist="gamma", method="ML",
                                                   fitkwargs={"floc": 0})
    assert isinstance(out, mx.DataArray) and out.dims == ("time", "lat", "lon") and out.values.shape == (36, 2, 3)
    np.testing.assert_array_equal(np.asarray(out.coords["lat"].values), np.arange(2) * 0.25)
    assert str(np.asarray(out.coords["time"].values)[1]) == "1981-02-01"
    params = stats.standardized_index_fit_params(da, freq="MS", window=3, dist="gamma", method="ML",
                                                 zero_inflated=True, fitkwargs={"floc": 0})
    assert isinstance(params, mx.DataArray) and params.coords["number_of_zeros"].dims == ("month", "lat", "lon")
    again = indices.standardized_precipitation_index(da, params=params)
    np.testing.assert_array_equal(np.asarray(again.values), np.asarray(out.values))


def test_device_outputs_option(host):
    from xclim_b200 import indices
    from xclim_b200.options import set_options
    da = _field(_pr(365 * 2, seed=5))
    with set_options(device_outputs=True):
        out = indices.standardized_precipitation_index(da, window=2, fitkwargs={"floc": 0})
    assert isinstance(out.values, torch.Tensor) and out.values.dtype == torch.float64
    ref = indices.standardized_precipitation_index(da, window=2, fitkwargs={"floc": 0})
    np.testing.assert_array_equal(out.values.numpy(), ref.values)


def test_errors(host):
    from xclim_b200 import indices, stats
    da = _field(_pr(365 * 3, seed=1))
    spi = indices.standardized_precipitation_index
    with pytest.raises(ValueError, match="Pass a value for `floc`"):
        spi(da, method="APP")
    with pytest.raises(NotImplementedError, match="Nelder-Mead"):
        spi(da)
    with pytest.raises(NotImplementedError, match="not yet implemented"):
        spi(da, dist="weibull_min", fitkwargs={"floc": 0})
    with pytest.raises(NotImplementedError, match="genextreme"):
        spi(da, dist="genextreme", fitkwargs={"floc": 0})
    with pytest.raises(NotImplementedError, match="APP method is not implemented for genextreme"):
        spi(da, dist="genextreme", method="APP", fitkwargs={"floc": 0})
    with pytest.raises(NotImplementedError, match="fisk ML"):
        spi(da, dist="fisk", fitkwargs={"floc": 0})
    with pytest.raises(NotImplementedError, match="fscale"):
        spi(da, fitkwargs={"floc": 0, "fscale": 1})
    with pytest.raises(NotImplementedError, match="weekly"):
        spi(da, freq="W", fitkwargs={"floc": 0})
    with pytest.raises(ValueError, match="frequency `YS`"):
        spi(da, freq="YS", fitkwargs={"floc": 0})
    with pytest.raises(ValueError, match="prob_zero_interpolation"):
        spi(da, fitkwargs={"floc": 0}, prob_zero_interpolation="lower")
    with pytest.raises(ValueError, match="plotting_position_zero"):
        spi(da, fitkwargs={"floc": 0}, plotting_position_zero="hazen")
    with pytest.raises(ValueError, match="must be given"):
        stats.standardized_index(da, "MS", None, "gamma", "ML", True, {"floc": 0}, None, None)
    with pytest.raises(NotImplementedError, match="rv_continuous"):
        stats.standardized_index_fit_params(da, "MS", 1, st.gamma, "APP", fitkwargs={"floc": 0})
    wb = _field(np.random.default_rng(0).normal(0, 1, (365 * 2, 1, 2)).astype(np.float32))
    with pytest.raises(ValueError, match="Maximum likelihood estimation with 'gamma'"):
        indices.standardized_precipitation_evapotranspiration_index(wb, fitkwargs={"floc": 0})
    # params of another calendar, legacy params
    p365 = stats.standardized_index_fit_params(da, "D", 1, "gamma", "APP", True, {"floc": 0})
    std = _field(_pr(366 * 2, seed=3), start="1984-01-01", calendar="standard")
    with pytest.raises(NotImplementedError, match="another calendar"):
        indices.standardized_precipitation_index(std, params=p365)
    legacy = p365.assign_attrs()
    legacy.coords = {k: v for k, v in p365.coords.items() if k not in ("number_of_zeros", "number_of_notnull")}
    with pytest.raises(NotImplementedError, match="prob_of_zero"):
        indices.standardized_precipitation_index(da, params=legacy)


# ---- argument checks of the C entry points (host side, no device work)
@pytest.fixture(scope="module")
def lib():
    from xclim_b200 import _build, _lib
    if not os.path.exists(_build.LIB_PATH):
        _build.build()
    return _lib.load()


INVALID, UNSUPPORTED = -1, -2


def test_entry_point_argument_checks(lib):
    buf = (C.c_double * 64)()
    p = C.cast(buf, C.c_void_p)
    assert lib.xc_si_fit_workspace_bytes(10, 7) == 280 and lib.xc_si_fit_workspace_bytes(0, 7) == -1

    def fit(x=p, T=4, Cn=4, ldx=4, goff=p, steps=p, G=1, max_n=4, dist=0, method=0, zi=1, floc=0.0, params=p,
            nz=p, nn=p, status=p, ws=p, wsb=64):
        return lib.xc_si_fit_f32(x, T, Cn, ldx, goff, steps, G, max_n, dist, method, zi, floc, params, nz, nn, status,
                                 ws, wsb, None)

    for kw in ({"x": None}, {"goff": None}, {"steps": None}, {"params": None}, {"status": None}, {"ws": None}):
        assert fit(**kw) == INVALID and b"null pointer" in lib.xc_last_error(), kw
    assert fit(nz=None) == INVALID and b"n_zeros" in lib.xc_last_error()
    for kw in ({"T": 0}, {"Cn": 0}, {"ldx": 3}):
        assert fit(**kw) == INVALID and b"shape" in lib.xc_last_error(), kw
    assert fit(G=0) == INVALID and b"group" in lib.xc_last_error()
    assert fit(wsb=63) == INVALID and b"workspace too small" in lib.xc_last_error()
    assert fit(floc=float("nan")) == INVALID and b"floc" in lib.xc_last_error()
    assert fit(dist=3) == INVALID and b"distribution" in lib.xc_last_error()
    assert fit(method=2) == INVALID and b"method" in lib.xc_last_error()
    assert fit(dist=1, method=1) == UNSUPPORTED and b"fisk ML" in lib.xc_last_error()

    def apply(x=p, T=4, Cn=4, ldx=4, gos=p, G=1, params=p, nz=p, nn=p, dist=0, zi=1, out=p, ldo=4):
        return lib.xc_si_apply_f32(x, T, Cn, ldx, gos, G, params, nz, nn, dist, zi, 1.0, 0.0, 1.0, out, ldo, None)

    for kw in ({"x": None}, {"gos": None}, {"params": None}, {"out": None}):
        assert apply(**kw) == INVALID and b"null pointer" in lib.xc_last_error(), kw
    assert apply(nn=None) == INVALID and b"n_notnull" in lib.xc_last_error()
    for kw in ({"T": 0}, {"ldx": 3}, {"ldo": 3}):
        assert apply(**kw) == INVALID and b"shape" in lib.xc_last_error(), kw
    for G in (0, 32768):
        assert apply(G=G) == INVALID and b"group" in lib.xc_last_error()
    assert apply(dist=5) == INVALID and b"distribution" in lib.xc_last_error()
    assert apply(T=65535 * 16 + 1) == INVALID and b"longer" in lib.xc_last_error()

    def roll(x=p, T=4, Cn=4, ldx=4, w=2, out=p, ldo=4):
        return lib.xc_rolling_mean_f32(x, T, Cn, ldx, w, out, ldo, None)

    assert roll(x=None) == INVALID and b"null pointer" in lib.xc_last_error()
    assert roll(ldo=3) == INVALID and b"shape" in lib.xc_last_error()
    assert roll(w=0) == INVALID and b"window" in lib.xc_last_error()
    assert roll(T=65535 * 32 + 1) == INVALID and b"longer" in lib.xc_last_error()
