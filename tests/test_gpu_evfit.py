"""Frequency analysis on the GPU: the fit and transform kernels against the host build of the same device code
(tests/csrc/evfit_host.cpp), and frequency_analysis end to end against the oracle by the likelihood rule."""
import os
import sys
import warnings

import numpy as np
import pytest
import scipy.stats as st

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import evfit_host_build as H  # noqa: E402
from oracle import evfit_oracle as O  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore::RuntimeWarning")]
GOLD = np.load(os.path.join(HERE, "golden", "ref_evfit.npz"))


def _torch():
    import torch
    return torch


def _gev_grid(C, n, seed):
    rng = np.random.default_rng(seed)
    c = rng.uniform(-0.4, 0.3, C)
    loc = rng.uniform(-50, 400, C)
    scale = rng.uniform(0.5, 80, C)
    return st.genextreme.rvs(c, loc=loc, scale=scale, size=(n, C), random_state=rng).astype(np.float32)


def _compare(dev, host, dist):
    """norm bit for bit; gumbel_r / genextreme at 1e-12 relative (the GEV shape, dimensionless and often near
    0, at 1e-12 absolute): the device's exp / log1p may differ from the host libm's by an ulp."""
    if dist == "norm":
        np.testing.assert_array_equal(dev, host)
        return
    np.testing.assert_array_equal(np.isnan(dev), np.isnan(host))
    if dist == "genextreme":
        np.testing.assert_allclose(dev[0], host[0], rtol=0, atol=1e-12)
        dev, host = dev[1:], host[1:]
    np.testing.assert_allclose(dev, host, rtol=1e-12, atol=0)


@pytest.mark.parametrize("dist", ["norm", "gumbel_r", "genextreme"])
@pytest.mark.parametrize("C,n", [(1, 30), (127, 60), (128, 150), (129, 30), (1000, 150)])
def test_fit_kernel_against_host_build(dist, C, n):
    from xclim_b200 import _lib, device
    torch = _torch()
    x = _gev_grid(C, n, C + n)
    x[::7, ::3] = np.nan
    x[3, ::5] = np.inf
    p, status = device.ev_fit(torch.from_numpy(x).cuda(), _lib.EV_DISTS[dist])
    ph, sh = H.fit(x, dist)
    assert status == sh == 0
    _compare(p.cpu().numpy(), ph, dist)


@pytest.mark.parametrize("dist", ["norm", "gumbel_r", "genextreme"])
def test_fit_kernel_hostile_samples_and_views(dist):
    """The golden samples (edges, ties, constants, non-finite, 1e-30 / 1e30) as columns of an ldx > C view."""
    from xclim_b200 import _lib, device
    torch = _torch()
    X = GOLD["x"].T.copy()                    # (300, cases)
    wide = np.full((X.shape[0], X.shape[1] + 37), 5.0, np.float32)
    wide[:, 11:11 + X.shape[1]] = X
    view = torch.from_numpy(wide).cuda()[:, 11:11 + X.shape[1]]
    assert view.stride(0) > view.shape[1]
    p, status = device.ev_fit(view, _lib.EV_DISTS[dist])
    ph, sh = H.fit(X, dist)
    assert status == sh
    _compare(p.cpu().numpy(), ph, dist)


@pytest.mark.parametrize("dist", ["norm", "gumbel_r", "genextreme"])
@pytest.mark.parametrize("kind", ["ppf", "isf", "cdf"])
def test_transform_kernel_against_host_build(dist, kind):
    from xclim_b200 import _lib, device
    torch = _torch()
    x = _gev_grid(300, 60, 9)
    ph, _ = H.fit(x, dist)
    ph[:, 5] = np.nan
    q = np.array([-1e3, 0.0, 25.0, 300.0]) if kind == "cdf" else np.array([0.0, 1e-9, 0.01, 0.5, 0.9, 0.99, 1.0])
    out = device.ev_transform(torch.from_numpy(ph).cuda(), _lib.EV_DISTS[dist], _lib.EV_KINDS[kind], q)
    want = H.transform(ph, dist, kind, q)
    got = out.cpu().numpy()
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    ok = np.isfinite(want)
    big = ok & (np.abs(np.where(ok, want, 0)) > 1e-20)
    np.testing.assert_allclose(got[big], want[big], rtol=1e-13, atol=0)
    # far tails (CDF values below 1e-20): the device and host exp / log1p differ by an ulp, amplified by exp(-exp)
    np.testing.assert_allclose(got[ok & ~big], want[ok & ~big], rtol=1e-11, atol=0)


@pytest.mark.parametrize("calendar", ["noleap", "standard"])
def test_frequency_analysis_end_to_end(calendar, monkeypatch):
    from xclim_b200 import stats
    from xclim_b200.field import Field
    from xclim_b200.options import OPTIONS
    from xclim_b200.timeaxis import TimeAxis
    rng = np.random.default_rng(11)
    years, Cx, Cy = 40, 4, 6
    ta = TimeAxis.daily("1981-01-01", 1, calendar)
    T = sum(366 if (calendar == "standard" and (y % 4 == 0 and (y % 100 != 0 or y % 400 == 0))) else 365
            for y in range(1981, 1981 + years))
    ta = TimeAxis.daily("1981-01-01", T, calendar)
    q = rng.gamma(2.0, 30.0, (T, Cx, Cy)).astype(np.float32)
    q[:, 0, 0] = np.nan
    da = Field(q, ("time", "x", "y"), ta, {}, {"units": "m3 s-1"})
    out = stats.frequency_analysis(da, mode="max", t=[2, 10, 100], dist="genextreme", window=3, freq="YS")
    assert out.dims == ("return_period", "x", "y") and out.attrs["units"] == "m3 s-1"
    got = np.asarray(out.values)
    assert np.isnan(got[:, 0, 0]).all() and np.isfinite(got.reshape(3, -1)[:, 1:]).all()
    # the same extremes restated on the host, fitted by the oracle
    roll = np.lib.stride_tricks.sliding_window_view(q.astype(np.float64), 3, axis=0).mean(-1).astype(np.float32)
    y = ta.year[2:]
    ext = np.stack([roll[y == yy].max(0) for yy in range(1981, 1981 + years)])
    ext[0] = np.maximum(ext[0], -np.inf)
    for c in range(1, Cx * Cy):
        i, j = divmod(c, Cy)
        v = ext[:, i, j]
        po = O.fit(v, "genextreme")
        pd = np.asarray(stats.fit(Field(ext[:, i:i + 1, j], ("time", "x"), None, {}, {}), "genextreme").values)
        fo = O.gev_nnlf(po, v)
        assert O.gev_nnlf(pd[:, 0], v) <= fo + 1e-9 * max(1, abs(fo))
        np.testing.assert_allclose(got[:, i, j], O.return_levels(po[:, None], "genextreme", (2, 10, 100))[:, 0],
                                   rtol=1e-4)
    # host-backed input above the streaming threshold takes the slab streamer and gives the same result
    monkeypatch.setitem(OPTIONS, "stream_min_bytes", 1 << 10)
    monkeypatch.setitem(OPTIONS, "stream_slab_bytes", q.nbytes // 3)
    out_s = stats.frequency_analysis(da, mode="max", t=[2, 10, 100], dist="genextreme", window=3, freq="YS")
    np.testing.assert_array_equal(np.asarray(out_s.values), got)


@pytest.mark.parametrize("n", [30, 60, 150])
def test_realistic_grid_converges(n):
    """Zero NaN cells on realistic GEV samples (c in [-0.4, 0.3]).  Small samples can still have their only
    likelihood optimum beyond c = 1 (scipy's simplex then stops at c > 1); those are NaN by design."""
    from xclim_b200 import _lib, device
    torch = _torch()
    rng = np.random.default_rng(21 + n)
    C = 4096
    c, loc, scale = rng.uniform(-0.4, 0.3, C), rng.uniform(-50, 400, C), rng.uniform(0.5, 80, C)
    x = st.genextreme.rvs(c, loc=loc, scale=scale, size=(n, C), random_state=rng).astype(np.float32)
    p, status = device.ev_fit(torch.from_numpy(x).cuda(), _lib.EV_DISTS["genextreme"])
    assert status == 0 and torch.isfinite(p).all()
    _compare(p.cpu().numpy(), H.fit(x, "genextreme")[0], "genextreme")
