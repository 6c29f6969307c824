"""Detrended quantile mapping and generic.detrend without a GPU: the oracle (oracle/dqm_oracle.py) on known answers
and against its kernel-basis form, the monotone-transform argument behind training on the raw series, the host
wrappers sdba.DetrendedQuantileMapping and generic.detrend over stand-ins defined here, and the argument validation
of the new C entry points through the real library."""
import ctypes as C

import numpy as np
import pytest
import torch

import fake_device
from oracle import dqm_oracle as D
from oracle import xclim_oracle as O
from xb_helpers import make_field


# ---- oracle known answers
def test_linear_series_detrends_to_zero():
    T = 500
    t = np.arange(T)
    y = np.stack([3 + 0.05 * t, 280 - 0.01 * t, 1e3 + 0.3 * t], axis=1).astype(np.float32)
    for deg in (1, 2):
        r = D.detrend(y, deg, start_ns=11 * 365 * D.NS_PER_DAY)
        assert r.dtype == np.float64
        # what is left is the float32 rounding of the line (half an ulp of ~1150 is 6e-5)
        assert np.abs(r).max() < 2e-4


def test_degree_zero_is_mean_removal():
    rng = np.random.default_rng(1)
    y = (280 + 5 * rng.standard_normal((300, 4))).astype(np.float32)
    y[rng.random(y.shape) < 0.1] = np.nan
    r = D.detrend(y, 0)
    np.testing.assert_allclose(r, y.astype(np.float64) - np.nanmean(y.astype(np.float64), axis=0), rtol=0, atol=1e-9)
    assert np.array_equal(np.isnan(r), np.isnan(y))


def test_few_valid_steps_and_all_nan():
    T = 50
    y = np.full((T, 4), np.nan, np.float32)
    y[7, 0] = 4.0                         # one valid step, degree 2 -> the constant through it
    y[[3, 40], 1] = [1.0, 9.0]            # two valid steps, degree 2 -> the line through them
    y[:, 3] = np.arange(T, dtype=np.float32)
    y[5, 3] = np.inf                      # an infinite value: the whole cell is NaN (not pinned against xarray)
    tr = D.poly_trend(y, 2)
    assert abs(tr[7, 0] - 4.0) < 1e-9
    np.testing.assert_allclose(tr[[3, 40], 1], [1.0, 9.0], rtol=0, atol=1e-8)
    assert np.isnan(tr[:, 2]).all() and np.isnan(tr[:, 3]).all()
    r = D.detrend(y, 2)
    assert np.array_equal(np.isnan(r[:, :2]), np.isnan(y[:, :2]))


@pytest.mark.parametrize("kind", ["+", "*"])
def test_ref_is_hist_gives_identity_factors(kind):
    rng = np.random.default_rng(2)
    x = (5 + rng.gamma(2.0, 2.0, (400, 6))).astype(np.float32)
    x[rng.random(x.shape) < 0.05] = np.nan
    af, hq, sc = D.dqm_train(x, x, 15, kind)
    assert np.all(af == (0 if kind == "+" else 1))
    assert np.all(sc == (0 if kind == "+" else 1))
    assert af.dtype == hq.dtype == sc.dtype == np.float32


def test_train_restates_eqm_on_normalised_series():
    rng = np.random.default_rng(3)
    ref = (285 + 6 * rng.standard_normal((365, 5))).astype(np.float32)
    hist = (287 + 7 * rng.standard_normal((365, 5))).astype(np.float32)
    af, hq, sc = D.dqm_train(ref, hist, 12, "+")
    mr = np.float32(np.sum(ref[:, 2].astype(np.float64)) / 365)
    mh = np.float32(np.sum(hist[:, 2].astype(np.float64)) / 365)
    assert sc[2] == np.float32(mr - mh)
    e_af, e_hq = O.eqm_train((ref - mr).astype(np.float32)[:, 2:3], (hist - mh).astype(np.float32)[:, 2:3], 12, "+")
    np.testing.assert_array_equal(af[:, 2], e_af[:, 0])
    np.testing.assert_array_equal(hq[:, 2], e_hq[:, 0])


def _u_fit(y, deg):
    """Least squares in the kernel basis (numpy lstsq on the valid steps): (deg + 1, C) coefficients, row k = u^k."""
    T, Cn = y.shape
    u = D.basis_u(T)
    coef = np.zeros((deg + 1, Cn))
    for c in range(Cn):
        ok = ~np.isnan(y[:, c])
        V = np.vander(u[ok], deg + 1, increasing=True)
        coef[:, c] = np.linalg.lstsq(V, y[ok, c].astype(np.float64), rcond=None)[0]
    return coef


@pytest.mark.parametrize("deg", [0, 1, 2])
def test_kernel_basis_trend_matches_lstsq_trend(deg):
    rng = np.random.default_rng(4 + deg)
    T = 3650
    t = np.arange(T)
    y = (280 + 0.001 * t[:, None] + 8 * np.sin(2 * np.pi * t / 365)[:, None]
         + 3 * rng.standard_normal((T, 5))).astype(np.float32)
    y[rng.random(y.shape) < 0.03] = np.nan
    a = D.trend_from_coef(_u_fit(y, deg), T)
    b = D.poly_trend(y, deg, start_ns=4018 * D.NS_PER_DAY)
    assert np.abs(a - b).max() <= 1e-9 * np.nanmax(np.abs(y))


# ---- the monotone-transform argument (order statistics of the normalised series)
def _hostile_columns(rng):
    T = 257
    cols = [
        np.round(rng.gamma(0.5, 4.0, T) * 2) / 2,                              # ties, many zeros
        np.where(rng.random(T) < 0.5, -0.0, 0.0),                              # signed zeros
        np.where(rng.random(T) < 0.1, np.inf, 10 * rng.standard_normal(T)),   # +inf among ordinary values
        np.where(rng.random(T) < 0.1, -np.inf, 10 * rng.standard_normal(T)),
        np.where(rng.random(T) < 0.5, np.float32(3e38), np.float32(-3e38)),   # +-3e38
        -5 + rng.standard_normal(T),                                          # negative mean
        rng.standard_normal(T) * 1e-3,
    ]
    x = np.stack(cols, axis=1).astype(np.float32)
    x[rng.random(x.shape) < 0.05] = np.nan
    return x


def _order_stats(v):
    return np.sort(v[~np.isnan(v)], kind="stable")


def test_monotone_transform_commutes_with_order_statistics():
    """float32 rounding is monotone: for "+" with a finite constant and "*" with a finite positive one, x -> x (+) c
    is non-decreasing and never makes a NaN, so the sorted normalised series is the normalised sorted series and the
    EQM quantiles of the normalised series are the lerp of the normalised order statistics."""
    rng = np.random.default_rng(5)
    x = _hostile_columns(rng)
    consts = {"+": [np.float32(-285.3), np.float32(0.0), np.float32(-0.0), np.float32(3e38), np.float32(-1e-40)],
              "*": [np.float32(0.003), np.float32(1.0), np.float32(7.5), np.float32(3e-39), np.float32(1e30)]}
    nodes = O.eqm_nodes(20).astype(np.float32).astype(np.float64)
    for kind, cs in consts.items():
        for c in cs:
            for j in range(x.shape[1]):
                v = x[:, j]
                n_v = D._apply(v, c, kind)
                assert np.array_equal(np.isnan(n_v), np.isnan(v)), (kind, c, j)     # no NaN made
                s_raw, s_n = _order_stats(v), _order_stats(n_v)
                np.testing.assert_array_equal(D._apply(s_raw, c, kind), s_n, err_msg=f"{kind} {c} {j}")
                # the EQM node positions: lerp of the transformed neighbours == quantile of the transformed series
                n = s_raw.size
                pos = nodes * (n - 1)
                lo = np.floor(pos).astype(int)
                hi = np.minimum(lo + 1, n - 1)
                a0, a1 = D._apply(s_raw[lo], c, kind), D._apply(s_raw[hi], c, kind)
                np.testing.assert_array_equal(a0, s_n[lo])
                np.testing.assert_array_equal(a1, s_n[hi])


def test_non_monotone_transforms_are_detected():
    """What the train kernels send to the one-cell path: "*" with a negative, zero or non-finite constant reverses
    the order or makes NaN (inf * 0), and "+" with an infinite constant makes NaN (inf - inf)."""
    v = np.array([-np.inf, -2.0, 0.0, 3.0, np.inf], np.float32)
    neg = D._apply(v, np.float32(-0.5), "*")
    assert not np.array_equal(np.sort(neg), neg)                    # order reversed
    assert np.isnan(D._apply(v, np.float32(0.0), "*")).any()       # inf * 0
    assert np.isnan(D._apply(v, np.float32(np.inf), "+")).any()    # -inf + inf
    assert np.isnan(D._apply(v, np.float32(np.inf), "*")).any()    # 0 * inf
    # a mean of zero or a subnormal mean has no finite inverse under "*"
    assert not np.isfinite(D._inv(np.float32(0.0), "*")) and not np.isfinite(D._inv(np.float32(1e-45), "*"))


# ---- host wrappers over stand-ins
def fake_dqm_train(ref2d, hist2d, nq, kind_code):
    af, hq, sc = D.dqm_train(ref2d.numpy(), hist2d.numpy(), int(nq), "+" if kind_code == 0 else "*")
    return tuple(torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)) for a in (af, hq, sc))


CALLS = []


def fake_dqm_adjust(sim2d, af, hq, scaling, kind_code, interp_code, degree, want_coef=False):
    CALLS.append(degree)
    out = D.dqm_adjust(sim2d.numpy(), af.numpy(), hq.numpy(), scaling.numpy(), "+" if kind_code == 0 else "*",
                       "linear" if interp_code == 1 else "nearest", detrend=degree)
    return torch.from_numpy(out)


def fake_detrend(x2d, degree):
    return torch.from_numpy(D.detrend(x2d.numpy(), degree))


@pytest.fixture
def host(monkeypatch):
    fake_device.install(monkeypatch)
    from xclim_b200 import device
    monkeypatch.setattr(device, "dqm_train", fake_dqm_train)
    monkeypatch.setattr(device, "dqm_adjust", fake_dqm_adjust)
    monkeypatch.setattr(device, "detrend", fake_detrend)


def _series(seed, T=730, shape=(2, 3)):
    rng = np.random.default_rng(seed)
    ref = (285 + 6 * rng.standard_normal((T,) + shape)).astype(np.float32)
    hist = (286.5 + 7 * rng.standard_normal((T,) + shape)).astype(np.float32)
    sim = (288.5 + 7 * rng.standard_normal((T + 365,) + shape) + np.linspace(0, 3, T + 365)[:, None, None])
    return ref, hist, sim.astype(np.float32)


def test_dqm_host_wrapper(host):
    import xclim_b200
    from xclim_b200 import sdba
    ref, hist, sim = _series(9)
    f = lambda a: make_field(a, "1981-01-01", calendar="noleap", units="K")  # noqa: E731
    dqm = sdba.DetrendedQuantileMapping.train(f(ref), f(hist), nquantiles=15, kind="+", group="time")
    assert isinstance(dqm, sdba.EmpiricalQuantileMapping)
    ds = dqm.ds
    assert set(ds) == {"af", "hist_q", "scaling"}
    e_af, e_hq, e_sc = D.dqm_train(ref, hist, 15, "+")
    np.testing.assert_array_equal(ds["af"].values, e_af)
    np.testing.assert_array_equal(ds["hist_q"].values, e_hq)
    np.testing.assert_array_equal(ds["scaling"].values, e_sc)
    assert ds["scaling"].dims == ("d0", "d1") and ds["af"].dims == ("quantiles", "d0", "d1")
    for detrend, deg in ((1, 1), (0, 0), (2, 2), (True, 1), (False, 0), (np.int64(2), 2)):
        CALLS.clear()
        scen = dqm.adjust(f(sim), interp="linear", detrend=detrend)
        assert CALLS == [deg]
        exp = D.dqm_adjust(sim, e_af, e_hq, e_sc, "+", "linear", detrend=deg)
        np.testing.assert_array_equal(scen.values, exp)
    assert scen.values.dtype == np.float32 and scen.values.shape == sim.shape
    assert scen.attrs["units"] == "K" and scen.dims == f(sim).dims
    with xclim_b200.set_options(sdba_extra_output=True):         # the option does not change DQM's return value
        assert not isinstance(dqm.adjust(f(sim)), dict)
    for bad in ({"detrend": 3}, {"detrend": -1}, {"detrend": object()}, {"detrend": 1.0}, {"interp": "cubic"},
                {"extrapolation": "nan"}, {"adapt_freq_thresh": "1 mm/d"}, {"jitter_under_thresh_value": "0.01 mm/d"}):
        with pytest.raises(NotImplementedError):
            dqm.adjust(f(sim), **bad)
    with pytest.raises(ValueError):
        dqm.adjust(f(sim[:, :1]))
    with pytest.raises(NotImplementedError):
        sdba.DetrendedQuantileMapping.train(f(ref), f(hist), group="time.month")
    with pytest.raises(NotImplementedError):
        sdba.DetrendedQuantileMapping.train(f(ref), f(hist), adapt_freq_thresh="1 mm/d")
    with pytest.raises(ValueError):
        sdba.DetrendedQuantileMapping.train(f(ref), f(hist), kind="-")


def test_generic_detrend_host(host):
    from xclim_b200 import generic
    rng = np.random.default_rng(12)
    x = (280 + np.linspace(0, 2, 400)[None, :, None] + rng.standard_normal((3, 400, 2))).astype(np.float32)
    x[0, 5, 1] = np.nan
    fld = make_field(np.moveaxis(x, 1, 0), "1990-01-01", units="K", long_name="tas")
    fld = type(fld)(x, ("lat", "time", "lon"), fld.time, {}, dict(fld.attrs), "tas")   # time not first
    out = generic.detrend(fld, deg=2)
    assert out.dims == ("lat", "time", "lon") and out.values.dtype == np.float64
    assert out.attrs == {"units": "K", "long_name": "tas"}
    exp = np.moveaxis(D.detrend(np.moveaxis(x, 1, 0), 2), 0, 1)
    np.testing.assert_array_equal(out.values, exp)
    assert np.isnan(out.values[0, 5, 1]) and np.isfinite(out.values).sum() == x.size - 1
    with pytest.raises(NotImplementedError):
        generic.detrend(fld, dim="lat")
    with pytest.raises(NotImplementedError):
        generic.detrend(fld, deg=3)
    with pytest.raises(NotImplementedError):
        generic.detrend({"tas": fld})                          # a Dataset-like mapping
    with pytest.raises(ValueError):
        generic.detrend(fld, deg=-1)


# ---- argument validation of the C entry points (host side, no device work)
@pytest.fixture(scope="module")
def lib():
    import os

    from xclim_b200 import _build, _lib
    if not os.path.exists(_build.LIB_PATH):
        _build.build()
    return _lib.load()


INVALID, UNSUPPORTED = -1, -2


def test_dqm_train_argument_validation(lib):
    buf = (C.c_float * 16)()
    p = C.cast(buf, C.c_void_p)
    ws_min = lib.xc_dqm_train_workspace_bytes(4, 4, 20)
    assert ws_min == 256 + 256 + lib.xc_eqm_train_workspace_bytes(4, 4, 20)
    assert lib.xc_dqm_train_workspace_bytes(10950, 259200, 20) == \
        256 + 8 * 259200 + lib.xc_eqm_train_workspace_bytes(10950, 259200, 20)

    def call(ref=p, hist=p, T=4, Cn=4, ldx=4, nq=20, kind=0, af=p, hq=p, sc=p, ws=p, wsb=ws_min):
        return lib.xc_dqm_train_f32(ref, hist, T, Cn, ldx, nq, kind, af, hq, sc, ws, wsb, None)

    for kw in ({"ref": None}, {"hist": None}, {"af": None}, {"hq": None}, {"sc": None}, {"ws": None}):
        assert call(**kw) == INVALID and b"null pointer" in lib.xc_last_error(), kw
    for kw in ({"T": 0}, {"Cn": 0}, {"ldx": 3}):
        assert call(**kw) == INVALID and b"shape" in lib.xc_last_error(), kw
    for nq in (0, 65):
        assert call(nq=nq) == INVALID and b"[1, 64]" in lib.xc_last_error()
    assert call(kind=2) == INVALID and b"kind" in lib.xc_last_error()
    assert call(wsb=ws_min - 1) == INVALID and b"workspace too small" in lib.xc_last_error()
    assert call(T=32769, wsb=1 << 40) == UNSUPPORTED and b"32768" in lib.xc_last_error()


def test_poly_fit_adjust_detrend_argument_validation(lib):
    buf = (C.c_double * 16)()
    p = C.cast(buf, C.c_void_p)

    def fit(x=p, T=4, Cn=4, ldx=4, deg=1, kind=0, sc=None, coef=p):
        return lib.xc_poly_fit_f32(x, T, Cn, ldx, deg, kind, sc, coef, None)

    def adj(sim=p, T=4, Cn=4, ldx=4, af=p, hq=p, sc=p, coef=p, nq=20, kind=0, interp=1, deg=1, scen=p):
        return lib.xc_dqm_adjust_f32(sim, T, Cn, ldx, af, hq, sc, coef, nq, kind, interp, deg, scen, None)

    def det(x=p, T=4, Cn=4, ldx=4, coef=p, deg=1, out=p):
        return lib.xc_detrend_apply_f32(x, T, Cn, ldx, coef, deg, out, None)

    for fn, ptrs in ((fit, ("x", "coef")), (adj, ("sim", "af", "hq", "sc", "coef", "scen")), (det, ("x", "coef", "out"))):
        for k in ptrs:
            assert fn(**{k: None}) == INVALID and b"null pointer" in lib.xc_last_error(), (fn, k)
        for kw in ({"T": 0}, {"Cn": 0}, {"ldx": 3}):
            assert fn(**kw) == INVALID and b"shape" in lib.xc_last_error(), (fn, kw)
        for deg in (-1, 3):
            assert fn(deg=deg) == INVALID and b"degree" in lib.xc_last_error(), (fn, deg)
    assert fit(kind=2) == INVALID and b"kind" in lib.xc_last_error()
    assert adj(kind=2) == INVALID and b"kind" in lib.xc_last_error()
    assert adj(interp=2) == INVALID and b"interp" in lib.xc_last_error()
    for nq in (1, 201):
        assert adj(nq=nq) == INVALID and b"[2, 200]" in lib.xc_last_error()
