"""Frequency analysis on the CPU: the oracle (oracle/evfit_oracle.py) against the reference's own fits stored in
tests/golden/ref_evfit.npz, the host build of the device code (evfit_core.cuh) against the oracle and live scipy,
the reference tests' known answers, the host layer (xclim_b200/stats.py) over stand-in device functions, and the
argument checks of the C entry points.  The kernels themselves are checked by test_gpu_evfit.py.

Contracts (DESIGN s5): norm is bit for bit; gumbel_r is scipy's scale equation solved in float64 (scipy evaluates
it in float32 on float32 data, so against the stored reference it is compared by likelihood and return level);
genextreme is the optimum of the likelihood, compared by nnlf and by return levels, not by parameter bits.
Samples without a maximum of the likelihood (one repeated value; n <= 3 or a c >= 1 optimum for genextreme)
are NaN with a warning where the reference returns wherever its optimiser stopped."""
import ctypes as C
import os
import sys
import warnings

import numpy as np
import pytest
import scipy.stats as st
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import evfit_host_build as H  # noqa: E402
import fake_device  # noqa: E402
from oracle import evfit_oracle as O  # noqa: E402

pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")
GOLD = np.load(os.path.join(HERE, "golden", "ref_evfit.npz"))
NAMES = [str(s) for s in GOLD["names"]]
DISTS = [str(s) for s in GOLD["dists"]]
#: samples without a maximum of the likelihood: the reference returns where its optimiser stopped, we give NaN
NO_MAXIMUM = {"gumbel_r": {"constant", "constant_inexact"},
              "genextreme": {"n2", "n3", "n7", "constant", "constant_inexact"}}
#: scipy's float32 evaluation of the Gumbel scale equation overflows or loses the root on these
GUMBEL_F32_BROKEN = {"tiny", "huge"}
T_RL = (2, 10, 100)


def _sample(i):
    return GOLD["x"][i, :GOLD["n"][i]]


def _nnlf(dist, p, x):
    return float(getattr(st, dist).nnlf(p, O.finite(x).astype(np.float64)))


def _gold(dist, i):
    k = 3 if dist == "genextreme" else 2
    return GOLD["params"][DISTS.index(dist), i, :k]


def test_golden_provenance():
    assert str(GOLD["scipy_version"]) and (GOLD["error"] == 0).all()   # the reference raised on no case


@pytest.mark.parametrize("i", range(len(NAMES)), ids=NAMES)
def test_oracle_norm_exact(i):
    np.testing.assert_array_equal(O.fit(_sample(i), "norm"), _gold("norm", i))


@pytest.mark.parametrize("dist", ["gumbel_r", "genextreme"])
@pytest.mark.parametrize("i", range(len(NAMES)), ids=NAMES)
def test_oracle_against_reference(dist, i):
    x, ref = _sample(i), _gold(dist, i)
    name = NAMES[i]
    po = O.fit(x, dist)
    if len(O.finite(x)) <= 1:
        assert np.isnan(po).all() and np.isnan(ref).all()
        return
    if name in NO_MAXIMUM.get(dist, ()):
        # no maximum: the oracle is NaN or, still descending, below wherever the reference's optimiser stopped
        assert np.isnan(po).all() or _nnlf(dist, po, x) < _nnlf(dist, ref, x)
        assert np.isnan(H.fit(O.finite(x)[:, None], dist)[0]).all()
        return
    if dist == "gumbel_r" and name in GUMBEL_F32_BROKEN:
        assert not np.isfinite(ref).all() or abs(ref[1] / po[1] - 1) > 1e-3
        return
    if not np.isfinite(ref).all():          # the reference's optimiser left the float range (1e30 values)
        assert np.isfinite(po).all()
        return
    fo, fr = _nnlf(dist, po, x), _nnlf(dist, ref, x)
    assert fo <= fr + 1e-9 * max(1.0, abs(fr)), (fo, fr)
    if fo < fr - 1e-6 * max(1.0, abs(fr)):   # the reference stopped far from the optimum (1e-30 values)
        return
    rl_o, rl_r = O.return_levels(po[:, None], dist, T_RL), O.return_levels(ref[:, None], dist, T_RL)
    np.testing.assert_allclose(rl_o, rl_r, rtol=1e-4)


@pytest.mark.parametrize("i", range(len(NAMES)), ids=NAMES)
def test_oracle_gumbel_is_scipy_float64(i):
    x = O.finite(_sample(i))
    if x.size <= 1 or x.min() == x.max():
        return
    ref = np.array(st.gumbel_r.fit(x.astype(np.float64)))
    np.testing.assert_allclose(O.fit(x, "gumbel_r"), ref, rtol=1e-12, atol=1e-14 * max(1.0, abs(ref[1])))


@pytest.mark.parametrize("dist", DISTS)
def test_host_build_on_golden_samples(dist):
    X = GOLD["x"].T.copy()
    ph, status = H.fit(X, dist)
    for i, name in enumerate(NAMES):
        x, po = _sample(i), O.fit(_sample(i), dist)
        if dist == "norm":
            np.testing.assert_array_equal(ph[:, i], po, err_msg=name)
        elif np.isnan(po).all() or name in NO_MAXIMUM.get(dist, ()):
            assert np.isnan(ph[:, i]).all(), name
        elif dist == "gumbel_r":
            np.testing.assert_allclose(ph[:, i], po, rtol=1e-12, err_msg=name)
        else:
            fh, fo = _nnlf(dist, ph[:, i], x), _nnlf(dist, po, x)
            assert fh <= fo + 1e-12 * max(1.0, abs(fo)), (name, fh, fo)
            np.testing.assert_allclose(O.return_levels(ph[:, i:i + 1], dist, T_RL),
                                       O.return_levels(po[:, None], dist, T_RL), rtol=1e-6, err_msg=name)
    want = {"norm": 0, "gumbel_r": 2, "genextreme": 3}[dist]
    assert status == want


def _gev_grid(C, n, seed):
    rng = np.random.default_rng(seed)
    c = rng.uniform(-0.4, 0.3, C)
    x = np.stack([st.genextreme.rvs(ci, loc=30, scale=8, size=n, random_state=rng) for ci in c], 1)
    return x.astype(np.float32)


@pytest.mark.parametrize("n", [30, 60, 150])
def test_host_build_against_live_scipy(n):
    x = _gev_grid(48, n, n)
    x[5, 3] = np.nan
    x[7, 4] = np.inf
    pn, _ = H.fit(x, "norm")
    pg, sg = H.fit(x, "gumbel_r")
    pe, se = H.fit(x, "genextreme")
    assert sg == 0 and se == 0 and not np.isnan(pe).any()
    for c in range(x.shape[1]):
        v = O.finite(x[:, c])
        np.testing.assert_array_equal(pn[:, c], np.array(st.norm.fit(v), np.float64))
        np.testing.assert_allclose(pg[:, c], st.gumbel_r.fit(v.astype(np.float64)), rtol=1e-12)
        m, var = v.mean(), v.var()
        s = np.sqrt(6 * var) / np.pi
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ref = st.genextreme.fit(v, 0.1, loc=m - 0.57722 * s, scale=s)     # xclim's ML path
        fe, fr = _nnlf("genextreme", pe[:, c], v), _nnlf("genextreme", ref, v)
        assert fe <= fr + 1e-9 * max(1.0, abs(fr))
        np.testing.assert_allclose(O.return_levels(pe[:, c:c + 1], "genextreme", T_RL),
                                   O.return_levels(np.array(ref)[:, None], "genextreme", T_RL), rtol=1e-4)


def test_genextreme_known_answer():
    """tests/test_stats.py::test_genextreme_fit of the reference: (0.20949, 297.954091, 75.7911863) at 1e-5."""
    x = _sample(NAMES.index("ref_fixture"))
    want = (0.20949, 297.954091, 75.7911863)
    np.testing.assert_allclose(O.fit(x, "genextreme"), want, rtol=1e-5)
    np.testing.assert_allclose(H.fit(x[:, None], "genextreme")[0][:, 0], want, rtol=1e-5)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("kind", ["ppf", "isf", "cdf"])
def test_transforms_against_scipy(dist, kind):
    rng = np.random.default_rng(7)
    k = 3 if dist == "genextreme" else 2
    P = np.empty((k, 40))
    P[-2] = rng.uniform(-50, 50, 40)
    P[-1] = rng.uniform(0.1, 20, 40)
    if k == 3:
        P[0] = np.concatenate([rng.uniform(-0.6, 0.6, 34), [0.0, 1e-12, -1e-12, 1e-5, 0.9, -0.9]])
    P[-1, 0] = 0.0          # invalid scale
    P[-2, 1] = np.nan
    if kind == "cdf":
        q = np.array([-200.0, -10.0, 0.0, 3.5, 25.0, 80.0, 1e4, np.nan])
    else:
        q = np.array([0.0, 1e-300, 1e-12, 0.01, 0.5, 0.9, 0.99, 1 - 1e-12, 1.0, np.nan, -0.1, 1.5])
    got = H.transform(P, dist, kind, q)
    want = O.transform(P, dist, kind, q)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    ok = np.isfinite(want)
    np.testing.assert_array_equal(got[~ok & ~np.isnan(want)], want[~ok & ~np.isnan(want)])
    big = ok & (np.abs(np.where(ok, want, 0)) > 1e-20)
    np.testing.assert_allclose(got[big], want[big], rtol=1e-13)
    np.testing.assert_allclose(got[ok & ~big], want[ok & ~big], rtol=1e-12, atol=1e-300)   # far tails


# ---- the host layer over stand-in device functions
def fake_ev_fit(x2d, dist_code):
    p, s = H.fit(x2d.numpy(), {0: "norm", 1: "gumbel_r", 2: "genextreme"}[dist_code])
    return torch.from_numpy(p), s


def fake_ev_transform(params, dist_code, kind_code, q):
    return torch.from_numpy(H.transform(params.numpy(), {0: "norm", 1: "gumbel_r", 2: "genextreme"}[dist_code],
                                        {0: "ppf", 1: "isf", 2: "cdf"}[kind_code], q))


def fake_rolling_mean(x2d, window):
    from oracle import stdindex_oracle
    return torch.from_numpy(stdindex_oracle.rolling_mean(x2d.numpy(), int(window)))


@pytest.fixture
def host(monkeypatch):
    from xclim_b200 import device
    fake_device.install(monkeypatch)
    monkeypatch.setattr(device, "ev_fit", fake_ev_fit)
    monkeypatch.setattr(device, "ev_transform", fake_ev_transform)
    monkeypatch.setattr(device, "rolling_mean", fake_rolling_mean)


def _field(values, dims=("time", "x"), start="2001-01-01", calendar="noleap", units="m3 s-1"):
    from xclim_b200.field import Field
    from xclim_b200.timeaxis import TimeAxis
    ta = TimeAxis.daily(start, values.shape[dims.index("time")], calendar)
    return Field(values, dims, ta, {}, {"units": units, "standard_name": "discharge"})


def test_fit_container(host):
    from xclim_b200 import stats
    x = _gev_grid(5, 40, 1)
    x[:, 2] = np.nan
    x[:39, 3] = np.nan                               # one value left: NaN
    p = stats.fit(_field(x.T.copy(), dims=("x", "time")), "genextreme", method="MLE")
    assert p.dims == ("x", "dparams") and list(p.coords["dparams"]) == ["c", "loc", "scale"]
    assert np.isnan(p.values[2]).all() and np.isnan(p.values[3]).all() and np.isfinite(p.values[[0, 1, 4]]).all()
    assert p.attrs["original_units"] == "m3 s-1" and p.attrs["units"] == "" and p.attrs["scipy_dist"] == "genextreme"
    assert p.attrs["estimator"] == "Maximum likelihood" and p.attrs["method"] == "MLE"
    np.testing.assert_array_equal(p.values.T, H.fit(x, "genextreme")[0])
    pn = stats.fit(_field(x), "norm")
    assert pn.dims == ("dparams", "x") and list(pn.coords["dparams"]) == ["loc", "scale"]


def test_quantiles_cdf_and_fa(host):
    from xclim_b200 import stats
    x = _gev_grid(4, 50, 2)
    p = stats.fit(_field(x), "gumbel_r")
    q = stats.parametric_quantile(p, [0.9, 0.99])
    assert q.dims == ("quantile", "x") and q.attrs["units"] == "m3 s-1" and q.attrs["standard_name"] == "discharge"
    np.testing.assert_allclose(q.values, O.transform(np.asarray(p.values), "gumbel_r", "isf", [0.1, 0.01]),
                               rtol=1e-13)
    q2 = stats.parametric_quantile(p, [0.1, 0.99])                   # not all above 1/2: ppf
    np.testing.assert_allclose(q2.values, O.transform(np.asarray(p.values), "gumbel_r", "ppf", [0.1, 0.99]),
                               rtol=1e-13)
    c = stats.parametric_cdf(p, [20.0, 40.0])
    assert c.dims == ("cdf", "x") and list(c.coords["cdf"]) == [20.0, 40.0]
    r = stats.fa(_field(x), [2, 20], "gumbel_r", mode="min")
    assert r.dims == ("return_period", "x") and r.attrs["mode"] == "min"
    np.testing.assert_allclose(r.values, O.transform(np.asarray(p.values), "gumbel_r", "ppf", [0.5, 0.05]),
                               rtol=1e-13)


def test_frequency_analysis_host_layer(host):
    """test_frequency_analysis of the reference: shape, NaN cell, units and dims, time not first."""
    from xclim_b200 import stats
    rng = np.random.default_rng(3)
    q = rng.gamma(2.0, 30.0, (365 * 12, 2, 3)).astype(np.float32)
    q[:, 0, 0] = np.nan
    da = _field(q, dims=("time", "x", "y"))
    out = stats.frequency_analysis(da, mode="max", t=2, dist="genextreme", window=6, freq="YS")
    assert out.dims == ("return_period", "x", "y") and out.values.shape == (1, 2, 3)
    assert np.isnan(out.values[:, 0, 0]) and not np.isnan(out.values[:, 1, 1])
    assert out.attrs["units"] == "m3 s-1"
    tr = _field(np.ascontiguousarray(np.moveaxis(q, 0, -1)), dims=("x", "y", "time"))
    out2 = stats.frequency_analysis(tr, mode="max", t=2, dist="genextreme", window=6, freq="YS")
    assert out2.dims == ("return_period", "x", "y")   # the extremes, like every resampled output here, lead
    np.testing.assert_array_equal(out2.values, out.values)
    s = stats.frequency_analysis(da, mode="min", t=[2, 5], dist="norm", season="JJA")
    assert s.values.shape == (2, 2, 3) and s.attrs["mode"] == "min"


def test_default_freq():
    from xclim_b200 import generic
    assert generic.default_freq() == "YS-JAN"
    assert generic.default_freq(season="DJF") == "YS-DEC"
    assert generic.default_freq(month=[7, 8]) == "YS-JUL"
    assert generic.default_freq(doy_bounds=(60, 100)) == "YS-FEB"
    assert generic.default_freq(date_bounds=("04-15", "09-01")) == "YS-APR"
    with pytest.raises(ValueError, match="Unknown group"):
        generic.default_freq(hour=3)


def test_errors(host):
    from xclim_b200 import stats
    da = _field(_gev_grid(2, 20, 4))
    with pytest.raises(ValueError, match="Fitting method not recognized"):
        stats.fit(da, "norm", method="XYZ")
    with pytest.raises(ValueError, match="not found in scipy.stats"):
        stats.fit(da, "not_a_law")
    with pytest.raises(ValueError, match="PWM"):
        stats.fit(da, "genextreme", method="PWM")
    for method in ("MM", "APP", "MSE", "MPS"):
        with pytest.raises(NotImplementedError):
            stats.fit(da, "genextreme", method=method)
    with pytest.raises(NotImplementedError):          # test_fit / test_fa of the reference use lognorm
        stats.fit(da, "lognorm")
    with pytest.raises(NotImplementedError):
        stats.fa(da, 10, "lognorm")
    with pytest.raises(NotImplementedError):
        stats.fit(da, st.genextreme)
    with pytest.raises(NotImplementedError):
        stats.fit(da, "genextreme", dim="x")
    with pytest.raises(NotImplementedError):
        stats.fit(da, "genextreme", floc=0.0)
    with pytest.raises(ValueError, match="Mode"):
        stats.fa(da, 10, "norm", mode="middle")
    with pytest.raises(ValueError, match="Mode"):
        stats.frequency_analysis(da, mode="mean", t=10, dist="norm")
    p = stats.fit(da, "norm")
    with pytest.raises(ValueError, match="one-dimensional"):
        import mini_xarray as mx
        stats.parametric_cdf(p, mx.DataArray(np.zeros((2, 2)), dims=("a", "b")))


def test_no_maximum_warns(host):
    from xclim_b200 import stats
    x = _gev_grid(3, 30, 5)
    x[:, 1] = 7.0
    with pytest.warns(RuntimeWarning, match="1 cell"):
        p = stats.fit(_field(x), "genextreme")
    assert np.isnan(p.values[:, 1]).all() and np.isfinite(p.values[:, [0, 2]]).all()


# ---- argument checks of the C entry points (host side, no device work)
@pytest.fixture(scope="module")
def lib():
    from xclim_b200 import _build, _lib
    if not os.path.exists(_build.LIB_PATH):
        _build.build()
    return _lib.load()


def test_entry_point_argument_checks(lib):
    INVALID = -1
    buf = (C.c_double * 64)()
    p = C.cast(buf, C.c_void_p)
    assert lib.xc_ev_fit_workspace_bytes(10, 7) == 280 and lib.xc_ev_fit_workspace_bytes(0, 7) == -1

    def fit(x=p, T=4, Cn=4, ldx=4, dist=2, params=p, status=p, ws=p, wsb=64):
        return lib.xc_ev_fit_f32(x, T, Cn, ldx, dist, params, status, ws, wsb, None)

    for kw in ({"x": None}, {"params": None}, {"status": None}, {"ws": None}):
        assert fit(**kw) == INVALID and b"null pointer" in lib.xc_last_error(), kw
    for kw in ({"T": 0}, {"Cn": 0}, {"ldx": 3}):
        assert fit(**kw) == INVALID and b"shape" in lib.xc_last_error(), kw
    assert fit(dist=3) == INVALID and b"distribution" in lib.xc_last_error()
    assert fit(wsb=63) == INVALID and b"workspace too small" in lib.xc_last_error()

    def tr(params=p, Cn=4, dist=0, kind=0, q=p, nq=2, out=p):
        return lib.xc_ev_transform_f64(params, Cn, dist, kind, q, nq, out, None)

    for kw in ({"params": None}, {"q": None}, {"out": None}):
        assert tr(**kw) == INVALID and b"null pointer" in lib.xc_last_error(), kw
    assert tr(Cn=0) == INVALID and b"shape" in lib.xc_last_error()
    for nq in (0, 65536):
        assert tr(nq=nq) == INVALID and b"probabilities" in lib.xc_last_error()
    assert tr(dist=-1) == INVALID and b"distribution" in lib.xc_last_error()
    assert tr(kind=3) == INVALID and b"transform" in lib.xc_last_error()
