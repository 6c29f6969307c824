"""Standardized indices on the GPU: the fit and transform kernels against the host build of the same code and
against oracle/stdindex_oracle.py, and the public entry points end to end."""
import os
import sys

import numpy as np
import pytest
import scipy.stats as st

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import stdindex_host_build as H  # noqa: E402
from oracle import stdindex_oracle as O  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore::RuntimeWarning")]


def ml_shape_tol(a):
    """Tolerance of the gamma ML shape: brentq's xtol + rtol, plus the conditioning of the root of
    log(a) - psi(a) = s.  Both sides evaluate that difference to a few ulp of |log a| + |psi(a)| and its slope is
    1/a - psi'(a) ~ -1/(2 a^2), so any two float64 root finders may differ by that noise over the slope."""
    import scipy.special as sc
    a = np.asarray(a, np.float64)
    slope = np.abs(1.0 / a - sc.polygamma(1, a))
    noise = 8 * 2.2e-16 * (np.abs(np.log(a)) + np.abs(sc.digamma(a)))
    return 2e-12 + 4 * 2.2e-16 * np.abs(a) + noise / slope


def _series(seed, T, C):
    rng = np.random.default_rng(seed)
    y = rng.gamma(0.8, 30.0, (T, C)).astype(np.float32)
    y[rng.random((T, C)) < 0.15] = 0.0
    y[rng.random((T, C)) < 0.03] = np.nan
    y[:, 0] = 0.0
    y[:, 1] = np.nan
    y[5 % T, 2] = np.inf
    y[9 % T, 2] = -np.inf
    return y


@pytest.mark.parametrize("dist,method", [("gamma", "APP"), ("gamma", "ML"), ("fisk", "APP"), ("lognorm", "APP"),
                                         ("lognorm", "ML")])
@pytest.mark.parametrize("T,C,G", [(12, 5, 12), (360, 129, 12), (1200, 256, 12), (730, 33, 365)])
def test_kernels_against_host_build_and_oracle(dist, method, T, C, G):
    import torch
    from xclim_b200 import _lib, device
    y = _series(T + C, T, C)
    gos = np.arange(T) % G
    goff, steps = H.csr(gos, G)
    x = torch.from_numpy(y).cuda()
    p, nz, nn, stat = device.si_fit(x, goff, steps, _lib.SI_DISTS[dist], _lib.SI_METHODS[method], True, 0.0)
    ph, nzh, nnh, sth = H.fit(y, gos, G, dist, method, True, 0.0)
    assert stat == sth
    np.testing.assert_array_equal(nz.cpu().numpy(), nzh)
    np.testing.assert_array_equal(nn.cpu().numpy(), nnh)
    pd = p.cpu().numpy()
    np.testing.assert_array_equal(np.isnan(pd), np.isnan(ph))
    ok = ~np.isnan(ph)
    if method == "ML" and dist == "gamma":
        assert np.all(np.abs(pd - ph)[ok] <= 2e-12 + 1e-15 * np.abs(ph[ok]))
    else:
        np.testing.assert_array_equal(pd, ph)
    # a column slice (ldx > C) gives the same bits
    wide = torch.zeros((T, C + 7), dtype=torch.float32, device="cuda")
    wide[:, 3:3 + C] = x
    p2, _, _, _ = device.si_fit(wide[:, 3:3 + C], goff, steps, _lib.SI_DISTS[dist], _lib.SI_METHODS[method], True, 0.0)
    assert torch.equal(torch.nan_to_num(p2, 1234.5), torch.nan_to_num(p, 1234.5))
    si = device.si_apply(x, gos, p, nz, nn, _lib.SI_DISTS[dist]).cpu().numpy()
    sio = O.transform(y, gos, pd, dist, nz.cpu().numpy(), nn.cpu().numpy())
    np.testing.assert_array_equal(np.isnan(si), np.isnan(sio))
    good = ~np.isnan(sio)
    np.testing.assert_array_equal(np.abs(si[good]) == 8.21, np.abs(sio[good]) == 8.21)
    assert np.all(np.abs(si - sio)[good] * st.norm.pdf(sio[good]) <= 1e-13)


@pytest.mark.parametrize("window", [1, 3, 30])
def test_rolling_mean_against_oracle(window):
    import torch
    from xclim_b200 import device
    y = _series(window, 400, 130)
    y[100:110, 7] = np.nan
    out = device.rolling_mean(torch.from_numpy(y).cuda(), window).cpu().numpy()
    np.testing.assert_array_equal(out, O.rolling_mean(y, window))


def _field(values, start="1981-01-01", calendar="noleap"):
    from xclim_b200.field import Field
    from xclim_b200.timeaxis import TimeAxis
    ta = TimeAxis.daily(start, values.shape[0], calendar)
    return Field(values, ("time", "lat", "lon"), ta, {}, {"units": "mm/d"})


@pytest.mark.parametrize("calendar", ["noleap", "standard", "360_day"])
@pytest.mark.parametrize("freq,window", [("MS", 3), ("D", 30), (None, 1)])
def test_spi_end_to_end_and_params_round_trip(calendar, freq, window):
    import torch
    from xclim_b200 import _lib, device, indices, stats
    rng = np.random.default_rng(7)
    n_days = {"noleap": 365, "standard": 365, "360_day": 360}[calendar] * 12
    pr = rng.gamma(0.5, 6.0, (n_days, 3, 4)).astype(np.float32)
    pr[rng.random(pr.shape) < 0.4] = 0.0
    da = _field(pr, calendar=calendar)
    kw = dict(freq=freq, window=window, dist="gamma", method="ML", fitkwargs={"floc": 0},
              cal_start="1982-01-01", cal_end="1990-12-31")
    si = indices.standardized_precipitation_index(da, **kw)
    out = np.asarray(si.values)
    # the same computation step by step: the kernel's preprocessing, then the oracle fit and transform
    series, keep, cell_shape, _ = stats._preprocess(da, freq, window, {})
    y = series.y.cpu().numpy()
    if window > 1 and freq == "MS":
        poff = da.time.period_offsets("MS")
        m, _ = device.period_reduce(torch.from_numpy(pr.reshape(n_days, -1)).cuda(), poff, _lib.STATS["mean"])
        np.testing.assert_array_equal(y, O.rolling_mean(m.cpu().numpy(), window))
    gid = np.asarray(series.group)
    cal = stats._cal_slice(series, "1982-01-01", "1990-12-31")
    G = series.max_g
    po, nzo, nno = O.fit_groups(y, gid, G, cal, "gamma", "ML", True, 0.0, numpy_logs=False)
    present = np.unique(gid[cal])
    gos = np.where(np.isin(gid, present), gid, -1)
    ph, nzh, nnh, _ = H.fit(y, gid, G, "gamma", "ML", True, 0.0, cal)
    sio = O.transform(y, gos, ph, "gamma", nzh, nnh).reshape(out.shape)
    good = ~np.isnan(sio)
    np.testing.assert_array_equal(np.isnan(out), ~good)
    assert np.all(np.abs(out - sio)[good] * st.norm.pdf(sio[good]) <= 1e-13)
    # the ML shape within brentq's tolerance, loc exact, the float32 scale within one float32 ulp
    np.testing.assert_array_equal(np.isnan(ph), np.isnan(po))
    ok = ~np.isnan(po[:, 0])
    assert np.all(np.abs(ph[:, 0] - po[:, 0])[ok] <= ml_shape_tol(po[:, 0][ok]))
    np.testing.assert_array_equal(ph[:, 1], po[:, 1])
    s32 = po[:, 2][ok].astype(np.float32)
    assert np.all(np.abs(ph[:, 2][ok].astype(np.float32) - s32) <= np.spacing(s32))
    # fit first, then params=: bit-identical to the one-call result
    params = stats.standardized_index_fit_params(da.isel_time(slice(0, None)), freq=freq, window=window, dist="gamma",
                                                 method="ML", zero_inflated=True, fitkwargs={"floc": 0})
    assert params.dims[:2] == (("month" if freq == "MS" else "dayofyear"), "dparams")
    si2 = indices.standardized_precipitation_index(da, params=params)
    si1 = indices.standardized_precipitation_index(da, freq=freq, window=window, dist="gamma", method="ML",
                                                   fitkwargs={"floc": 0})
    np.testing.assert_array_equal(np.asarray(si2.values), np.asarray(si1.values))


def test_spei_fit_data_error_and_unsupported():
    from xclim_b200 import indices
    rng = np.random.default_rng(3)
    wb = (rng.normal(0.0, 2.0, (365 * 5, 2, 2))).astype(np.float32)
    da = _field(wb)
    with pytest.raises(ValueError, match="Maximum likelihood"):
        indices.standardized_precipitation_evapotranspiration_index(da, fitkwargs={"floc": 0})
    with pytest.raises(NotImplementedError):
        indices.standardized_precipitation_evapotranspiration_index(da)
    with pytest.raises(NotImplementedError):
        indices.standardized_precipitation_evapotranspiration_index(da, freq="W", fitkwargs={"floc": -50})
    out = indices.standardized_precipitation_evapotranspiration_index(da, dist="fisk", method="APP",
                                                                      fitkwargs={"floc": -50.0})
    assert np.asarray(out.values).dtype == np.float64 and np.asarray(out.values).shape == (60, 2, 2)
