"""Standardized indices on the CPU: the special functions and whole cells of the host build of
stdindex_core.cuh against scipy and oracle/stdindex_oracle.py, and the oracle against scipy's own fit."""
import os
import sys

import numpy as np
import pytest
import scipy.special as sc
import scipy.stats as st

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import stdindex_host_build as H  # noqa: E402
from oracle import stdindex_oracle as O  # noqa: E402

pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")


def ml_shape_tol(a):
    """Tolerance of the gamma ML shape: brentq's xtol + rtol, plus the conditioning of the root of
    log(a) - psi(a) = s.  Both sides evaluate that difference to a few ulp of |log a| + |psi(a)| and its slope is
    1/a - psi'(a) ~ -1/(2 a^2), so any two float64 root finders may differ by that noise over the slope."""
    import scipy.special as sc
    a = np.asarray(a, np.float64)
    slope = np.abs(1.0 / a - sc.polygamma(1, a))
    noise = 8 * 2.2e-16 * (np.abs(np.log(a)) + np.abs(sc.digamma(a)))
    return 2e-12 + 4 * 2.2e-16 * np.abs(a) + noise / slope


def test_gammainc_against_scipy():
    a = np.logspace(-3, 5, 60)[:, None]
    x = a * np.logspace(-6, 3, 80)[None, :]
    A, X = np.broadcast_arrays(a, x)
    got, ref = H.gammainc(A, X), sc.gammainc(A, X)
    m = ref >= 1e-300
    rel = np.abs(got - ref)[m] / ref[m]
    # deep in the lower tail P = exp(-a phi) with a phi up to 700, and phi = u - log1p(u) cancels about
    # tenfold for |u| near 1/2: a few ulp of phi are a relative 5e-15 * a phi of P, so the bound grows with -log P
    tol = 1e-13 + 5e-15 * np.maximum(0.0, -np.log(ref[m]))
    assert np.all(rel <= tol), (rel / tol).max()
    assert np.all(rel[ref[m] >= 1e-10] <= 1e-13)
    # far below the mode with a >= 10 (u = (x - a) / a rounds to -1 once x < a 2^-53): finite, and 0 or subnormal
    # exactly where scipy's value is
    a2 = np.array([10.0, 12.0, 12.0, 50.0, 1e3, 1e5, 12.0, 30.0])
    x2 = np.array([1e-30, 1e-28, 1e-26, 1e-10, 1e-3, 1.0, 0.5, 2.0])
    got2, ref2 = H.gammainc(a2, x2), sc.gammainc(a2, x2)
    assert np.all(np.isfinite(got2)) and np.all(got2 >= 0)
    assert np.all(np.abs(got2 - ref2) <= 1e-13 * ref2 + 1e-300)


def test_digamma_and_ndtri_against_scipy():
    x = np.logspace(-3, 4, 2000)
    got, ref = H.digamma(x), sc.digamma(x)
    near = np.abs(x - 1.4616321449683623) < 0.05
    assert np.all(np.abs(got - ref)[near] <= 1e-15)
    assert np.all((np.abs(got - ref) / np.abs(ref))[~near] <= 2e-14)
    p = np.concatenate([np.logspace(-300, -1, 2000), 1 - np.logspace(-16, -1, 500), np.linspace(0.01, 0.99, 999),
                        0.5 + np.logspace(-16, -2, 100)])
    assert np.all(np.abs(H.ndtri(p) - sc.ndtri(p)) <= 1e-14 * np.abs(sc.ndtri(p)))
    sub = np.array([1e-305, 2.2e-308, 1e-310, 1e-315, 1e-320, 5e-324])      # subnormal probabilities
    assert np.all(np.abs(H.ndtri(sub) - sc.ndtri(sub)) <= 1e-14 * np.abs(sc.ndtri(sub)))
    z = np.linspace(-37, 9, 3000)
    assert np.all(np.abs(H.ndtr(z) - sc.ndtr(z)) <= 1e-12 * sc.ndtr(z))


@pytest.mark.parametrize("n", [0, 1, 2, 7, 8, 9, 30, 127, 128, 129, 300, 1000, 4097])
def test_pairwise_mean_matches_numpy(n):
    v = np.random.default_rng(n).gamma(0.7, 3.0, n).astype(np.float32) * np.float32(1e3)
    if n:
        assert H.np_mean(v) == v.mean()
    else:
        assert np.isnan(H.np_mean(v))


def test_oracle_gamma_ml_matches_scipy_fit():
    rng = np.random.default_rng(5)
    for n in (2, 9, 30, 129):
        x = rng.gamma(1.3, 20.0, n).astype(np.float32)
        a, loc, scale = st.gamma.fit(x, floc=0)
        p = O.fit_sample(x, "gamma", "ML", 0.0, numpy_logs=True)
        assert p[0] == a and p[2] == np.float64(scale)
        x2 = rng.lognormal(1.0, 0.8, n).astype(np.float32)
        s, _, sc_ = st.lognorm.fit(x2, floc=0)
        p2 = O.fit_sample(x2, "lognorm", "ML", 0.0, numpy_logs=True)
        assert p2[0] == np.float64(s) and p2[2] == np.float64(sc_)


def _samples(rng, T, C):
    y = rng.gamma(0.8, 30.0, (T, C)).astype(np.float32)
    y[rng.random((T, C)) < 0.15] = 0.0
    y[rng.random((T, C)) < 0.03] = np.nan
    y[:, 0] = 0.0                                  # a desert cell
    y[:, 1] = np.nan                               # an all-NaN cell
    y[5, 2], y[9, 2] = np.inf, -np.inf
    y[::7, 3] = np.float32(1e-30)
    return y


@pytest.mark.parametrize("dist,method", [("gamma", "APP"), ("gamma", "ML"), ("fisk", "APP"), ("lognorm", "APP"),
                                         ("lognorm", "ML")])
@pytest.mark.parametrize("zi", [True, False])
@pytest.mark.parametrize("years", [1, 4, 30, 140])
def test_host_build_cells_against_oracle(dist, method, zi, years):
    rng = np.random.default_rng(years * 7 + len(dist))
    T, C, G = 12 * years, 9, 12
    y = _samples(rng, T, C)
    if method == "ML" and not zi:
        y = np.where(y == 0, np.float32(0.5), y)   # ML requires every value > floc
        y[:, 0] = np.float32(3.0) + np.arange(T, dtype=np.float32)
    gos = np.arange(T) % G
    p, nz, nn, stat = H.fit(y, gos, G, dist, method, zi, 0.0)
    try:
        po, nzo, nno = O.fit_groups(y, gos, G, slice(None), dist, method, zi, 0.0, numpy_logs=False)
    except O.FitDataError:
        assert stat & 1
        return
    except ValueError:
        assert stat & 6
        return
    assert stat == 0
    if zi:
        np.testing.assert_array_equal(nz, nzo)
        np.testing.assert_array_equal(nn, nno)
    np.testing.assert_array_equal(np.isnan(p), np.isnan(po))
    if method == "APP" or dist == "lognorm":
        np.testing.assert_array_equal(p, po)
    else:
        ok = ~np.isnan(po[:, 0])
        assert np.all(np.abs(p[:, 0][ok] - po[:, 0][ok]) <= ml_shape_tol(po[:, 0][ok]))
        np.testing.assert_array_equal(p[:, 1], po[:, 1])
        s32 = np.abs(p[:, 2][ok].astype(np.float32) - po[:, 2][ok].astype(np.float32))
        assert np.all(s32 <= np.spacing(po[:, 2][ok].astype(np.float32)))
    si = H.apply(y, gos, p, dist, nz, nn)
    sio = O.transform(y, gos, p, dist, nz, nn)
    np.testing.assert_array_equal(np.isnan(si), np.isnan(sio))
    ok = ~np.isnan(sio)
    np.testing.assert_array_equal(np.abs(si[ok]) == 8.21, np.abs(sio[ok]) == 8.21)
    assert np.all(np.abs(si - sio)[ok] * st.norm.pdf(sio[ok]) <= 1e-13)


@pytest.mark.parametrize("pp,interp", [("ecdf", 1.0), ("weibull", 0.5), ((0.3, 0.4), 0.25)])
def test_zero_inflation_known_answers(pp, interp):
    alpha, beta = {"ecdf": (0, 1), "weibull": (0, 0)}.get(pp, pp)
    T, G = 24, 12
    y = np.zeros((T, 2), np.float32)
    y[:, 1] = np.where(np.arange(T) < 12, 0.0, 5.0).astype(np.float32)
    y[13, 1] = 7.0
    gos = np.arange(T) % G
    p, nz, nn, _ = H.fit(y, gos, G, "gamma", "APP", True, 0.0)
    si = H.apply(y, gos, p, "gamma", nz, nn, interp, alpha, beta)
    assert np.all(np.isnan(p[:, :, 0]))
    r1 = (1 - alpha) / (2 + 1 - alpha - beta)
    rn = (2 - alpha) / (2 + 1 - alpha - beta)
    exp0 = sc.ndtri((1 - interp) * r1 + interp * rn) if (1 - interp) * r1 + interp * rn < 1 else 8.21
    np.testing.assert_allclose(si[:, 0], np.clip(exp0, -8.21, 8.21), rtol=1e-14)
    if pp == "ecdf":
        assert np.all(si[:, 0] == 8.21)


def test_fit_data_error_and_constant_samples():
    y = np.array([[1.0], [2.0], [-1.0], [3.0]], np.float32)
    gos = np.zeros(4, int)
    _, _, _, stat = H.fit(y, gos, 1, "gamma", "ML", False, 0.0)
    assert stat == 1
    yc = np.full((5, 1), 2.0, np.float32)
    p, _, _, stat = H.fit(yc, np.zeros(5, int), 1, "gamma", "APP", False, 0.0)
    assert stat == 0 and p[0, 0, 0] == np.inf and p[0, 2, 0] == 0.0
    with pytest.raises(ValueError):
        st.gamma.fit(yc[:, 0], floc=0)
    _, _, _, stat = H.fit(yc, np.zeros(5, int), 1, "gamma", "ML", False, 0.0)
    assert stat & 6


@pytest.mark.parametrize("dist,shape,x", [("lognorm", 0.1, 0.022), ("gamma", 12.0, 1e-27), ("gamma", 40.0, 1e-30),
                                          ("fisk", 12.0, 1e-27)])
def test_subnormal_and_zero_cdf_clip_to_the_lower_bound(dist, shape, x):
    """CDF values that underflow to subnormals or zero give -8.21, as norm.ppf then the clip do in the reference."""
    y = np.array([[x], [1.0]], np.float32)
    p = np.array([[[shape], [0.0], [1.0]]])
    got = H.apply(y, np.zeros(2, int), p, dist)
    exp = O.transform(y, np.zeros(2, int), p, dist)
    assert got[0, 0] == -8.21 and exp[0, 0] == -8.21
    assert abs(got[1, 0] - exp[1, 0]) * st.norm.pdf(exp[1, 0]) <= 1e-13
