"""Detrended quantile mapping and generic.detrend on the GPU against the oracle (oracle/dqm_oracle.py; PARITY UNPINNED
against xsdba itself).  af, hist_q and scaling bit for bit; the kernel's trend coefficients against the lstsq trend;
scen bit for bit against the oracle fed the kernel's coefficients, and within 1e-5 of the lstsq oracle (a nearest
factor may flip only where d sits within 1e-9 of a bound).  Both kinds and interpolations, degrees 0 to 2, nq 2 to
64, cells the train selection sends to the one-cell kernel, series lengths 1 to 40000, column slices and a sample of
the headline band."""
import numpy as np
import pytest

from oracle import dqm_oracle as D

pytestmark = pytest.mark.gpu

KIND = {"+": 0, "*": 1}
INTERP = {"nearest": 0, "linear": 1}


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _np(t):
    return t.cpu().numpy()


def _train_data(rng, T, C, kind):
    if kind == "+":
        ref = 285 + 6 * rng.standard_normal((T, C))
        hist = 286.5 + 7 * rng.standard_normal((T, C))
    else:
        ref = 0.2 + rng.gamma(0.8, 4.0, (T, C))
        hist = 0.2 + rng.gamma(0.7, 5.0, (T, C))
    ref, hist = ref.astype(np.float32), hist.astype(np.float32)
    hist[rng.random(hist.shape) < 0.01] = np.nan
    hist[:, 1] = np.round(hist[:, 1])                                   # ties
    ref[:, 0] = np.nan                                                  # untrainable cell
    return ref, hist


def _sim(rng, T, C, kind):
    t = np.linspace(0, 1, T)[:, None]
    if kind == "+":
        s = 288.5 + 7 * rng.standard_normal((T, C)) + 4 * t - 3 * t * t
    else:
        s = (0.2 + rng.gamma(0.7, 5.5, (T, C))) * (1 + 0.3 * t)
    s = s.astype(np.float32)
    s[rng.random(s.shape) < 0.01] = np.nan
    return s


def _nearest_bounds(hq, af):
    ok = ~(np.isnan(hq) | np.isnan(af))
    h = hq[ok] / np.float32(2.0)
    return (h[1:] + h[:-1]).astype(np.float64)


def _compare_lstsq(scen, sim, af, hq, sc, kind, interp, deg):
    """scen against the lstsq oracle at 1e-5 relative; with nearest, a factor flip is allowed only where d lies
    within 1e-9 relative of a bound.  Returns the number of flips."""
    exp = D.dqm_adjust(sim, af, hq, sc, kind, interp, detrend=deg)
    bad = ~np.isclose(scen, exp, rtol=1e-5, atol=0, equal_nan=True)
    if not bad.any():
        return 0
    assert interp == "nearest", f"linear {kind} deg={deg}: {bad.sum()} values beyond 1e-5"
    y = D._apply(sim, sc, kind)
    tau = D.poly_trend(y, deg)
    with np.errstate(all="ignore"):
        d = y - tau if kind == "+" else y * (1.0 / tau)
    for t, c in zip(*np.nonzero(bad)):
        bd = _nearest_bounds(hq[:, c], af[:, c])
        assert np.min(np.abs(d[t, c] - bd) / np.abs(bd)) <= 1e-9, (t, c, d[t, c])
    return int(bad.sum())


@pytest.mark.parametrize("nq", [2, 20, 64])
@pytest.mark.parametrize("kind", ["+", "*"])
def test_dqm_train_bit_identical(cuda, kind, nq):
    from xclim_b200 import device
    rng = np.random.default_rng(71 + nq)
    ref, hist = _train_data(rng, 1500, 96, kind)
    af, hq, sc = (_np(a) for a in device.dqm_train(_cuda(ref), _cuda(hist), nq, KIND[kind]))
    e_af, e_hq, e_sc = D.dqm_train(ref, hist, nq, kind)
    np.testing.assert_array_equal(sc, e_sc)
    np.testing.assert_array_equal(hq, e_hq)
    np.testing.assert_array_equal(af, e_af)
    assert np.isnan(af[:, 0]).all() and np.isnan(sc[0])
    af2, hq2, sc2 = (_np(a) for a in device.dqm_train(_cuda(hist), _cuda(hist), nq, KIND[kind]))
    ident = 0 if kind == "+" else 1
    assert ((af2 == ident) | (hq2 == 0)).all() and (sc2 == ident).all()      # "*": 0 / 0 where a quantile is 0


def _hostile_train(rng, T, kind):
    """64 cells (the cell-group kernel's layout), one hostile pattern in each of the first 16."""
    C = 64
    base = 5.0 if kind == "*" else 280.0
    x = (base + rng.gamma(2.0, 1.5, (T, C))).astype(np.float32)
    x[:, 0] = np.nan                                                    # all NaN
    x[:, 1] = 3.0                                                       # constant
    x[:, 2] = -(1 + rng.gamma(2.0, 1.0, T))                             # negative mean ("*": reversed order)
    x[:, 3] = rng.standard_normal(T)
    x[:, 3] -= np.float32(np.mean(x[:, 3].astype(np.float64)))          # mean near zero
    x[:, 4] = np.where(rng.random(T) < 0.5, np.float32(-0.0), np.float32(0.0))   # mean exactly zero
    x[:, 5] = np.round(rng.gamma(0.5, 4.0, T) * 2) / 2                  # ties, many zeros
    x[rng.random(T) < 0.1, 6] = np.inf                                  # +inf: infinite mean
    x[rng.random(T) < 0.1, 7] = -np.inf
    x[:, 8] = np.where(rng.random(T) < 0.5, np.float32(3e38), np.float32(-3e38))   # infinite range
    x[:, 9] = np.float32(1e-41) * rng.integers(1, 5, T)                 # subnormal mean
    x[:, 10] = np.float32(3e38) * rng.random(T).astype(np.float32)      # "*": a subnormal inverse
    x[rng.random(T) < 0.3, 11] = np.nan
    return x


# EQM's own limit (eqm.cu): a cell whose normalised values are infinite or span an infinite range is not supported
UNSUPPORTED = {"+": [6, 7, 8], "*": [6, 7, 8, 9]}


@pytest.mark.parametrize("kind", ["+", "*"])
def test_dqm_train_hostile_and_redo(cuda, kind, monkeypatch):
    """Cells whose normalisation is not a monotone map (mean <= 0, zero, subnormal or non-finite under "*", non-finite
    under "+") or whose range is infinite go from the cell-group kernel to the one-cell kernel.  The default dispatch
    and the one-cell kernel alone (XCLIM_B200_EQM_V1) agree bit for bit on every cell, and both match the oracle
    outside EQM's unsupported infinite ranges."""
    from xclim_b200 import device
    rng = np.random.default_rng(72)
    ref = _hostile_train(rng, 2000, kind)
    hist = _hostile_train(rng, 2000, kind)
    hist[:, 12:] *= np.float32(1.05)
    got = [_np(a) for a in device.dqm_train(_cuda(ref), _cuda(hist), 20, KIND[kind])]
    monkeypatch.setenv("XCLIM_B200_EQM_V1", "1")
    one = [_np(a) for a in device.dqm_train(_cuda(ref), _cuda(hist), 20, KIND[kind])]
    monkeypatch.delenv("XCLIM_B200_EQM_V1")
    for g, o, name in zip(got, one, ("af", "hist_q", "scaling")):
        np.testing.assert_array_equal(g.view(np.uint32), o.view(np.uint32), err_msg=f"paths {name}")
    exp = D.dqm_train(ref, hist, 20, kind)
    keep = np.setdiff1d(np.arange(64), UNSUPPORTED[kind])
    for g, e, name in zip(got, exp, ("af", "hist_q", "scaling")):
        np.testing.assert_array_equal(g[..., keep], e[..., keep], err_msg=f"oracle {name}")


@pytest.mark.parametrize("deg", [0, 1, 2])
@pytest.mark.parametrize("C", [37, 64])          # one cell per lane / four cells per lane
def test_poly_fit_against_lstsq(cuda, deg, C):
    from xclim_b200 import device
    rng = np.random.default_rng(73 + deg)
    T = 10950
    t = np.arange(T)
    y = (280 + 0.0004 * t[:, None] * rng.random(C) + 8 * np.sin(2 * np.pi * t / 365)[:, None]
         + 3 * rng.standard_normal((T, C))).astype(np.float32)
    y[rng.random(y.shape) < 0.02] = np.nan
    y[:, 0] = np.nan                                    # no valid step
    y[:, 1] = np.nan
    y[[100, 9000], 1] = [1.0, 5.0]                      # two valid steps
    y[:, 2] = np.nan
    y[4321, 2] = 7.5                                    # one valid step
    y[17, 3] = np.inf                                   # an infinite value
    coef = _np(device.poly_fit(_cuda(y), deg))
    assert coef.shape == (deg + 1, C) and coef.dtype == np.float64
    assert np.isnan(coef[:, [0, 3]]).all()
    tr = D.trend_from_coef(coef, T)
    ref = D.poly_trend(y, deg, start_ns=4018 * D.NS_PER_DAY)
    ok = ~np.isnan(y)
    err = np.where(ok, np.abs(tr - ref), 0.0).max(axis=0)[4:] / np.nanmax(np.abs(y[:, 4:]), axis=0)
    # reached on an H100: 2.2e-14 at most (degree 2)
    print(f"deg={deg} C={C}: max |trend - lstsq trend| / max|y| per cell = {err.max():.3e}")
    assert err.max() <= 1e-10
    assert abs(tr[4321, 2] - 7.5) <= 1e-12
    if deg >= 1:
        np.testing.assert_allclose(tr[[100, 9000], 1], [1.0, 5.0], rtol=1e-12)


@pytest.mark.parametrize("nq", [2, 20, 64])
@pytest.mark.parametrize("deg", [0, 1, 2])
@pytest.mark.parametrize("kind,interp", [("+", "linear"), ("+", "nearest"), ("*", "linear"), ("*", "nearest")])
def test_dqm_train_adjust(cuda, kind, interp, deg, nq):
    import xclim_b200  # noqa: F401
    from xclim_b200 import device, sdba
    from xb_helpers import make_field
    rng = np.random.default_rng(74 + nq + 10 * deg)
    T, C = 1500, 111
    ref, hist = _train_data(rng, T, C, kind)
    sim = _sim(rng, T + 400, C, kind)
    f = lambda a: make_field(a, "1981-01-01", calendar="noleap", units="K")  # noqa: E731
    dqm = sdba.DetrendedQuantileMapping.train(f(ref), f(hist), nquantiles=nq, kind=kind, group="time")
    ds = dqm.ds
    af, hq, sc = ds["af"].values, ds["hist_q"].values, ds["scaling"].values
    scen = dqm.adjust(f(sim), interp=interp, extrapolation="constant", detrend=deg).values
    _, coef = device.dqm_adjust(_cuda(sim), _cuda(af), _cuda(hq), _cuda(sc), KIND[kind], INTERP[interp], deg,
                                want_coef=True)
    exp = D.dqm_adjust(sim, af, hq, sc, kind, interp, detrend=deg, coef=_np(coef))
    np.testing.assert_array_equal(scen, exp)
    assert np.isnan(scen[:, 0]).all()
    flips = _compare_lstsq(scen, sim, af, hq, sc, kind, interp, deg)
    print(f"{kind} {interp} deg={deg} nq={nq}: nearest flips next to a bound: {flips}")


@pytest.mark.parametrize("kind", ["+", "*"])
def test_ref_is_hist_returns_sim(cuda, kind):
    from xclim_b200 import device
    rng = np.random.default_rng(75)
    ref, _ = _train_data(rng, 1200, 64, kind)
    ref[:, 0] = ref[:, 1]
    sim = _sim(rng, 1600, 64, kind)
    af, hq, sc = device.dqm_train(_cuda(ref), _cuda(ref), 20, KIND[kind])
    for interp in (0, 1):
        for deg in (0, 1, 2):
            scen = _np(device.dqm_adjust(_cuda(sim), af, hq, sc, KIND[kind], interp, deg))
            np.testing.assert_array_equal(scen, sim)


@pytest.mark.parametrize("T", [1, 2, 40, 10950, 40000])
def test_adjust_and_detrend_layouts(cuda, T):
    """Series lengths (adjust and detrend have no length limit), a column slice (ldx > C) and C not a multiple of 32:
    scen and detrend bit for bit against the oracle fed the kernel's coefficients, detrend close to the lstsq one."""
    from xclim_b200 import device, generic
    from xb_helpers import make_field
    rng = np.random.default_rng(76)
    C, nq = 70, 20
    big = (285 + 8 * rng.standard_normal((T, C + 9)) + np.linspace(0, 5, T)[:, None]).astype(np.float32)
    big[rng.random(big.shape) < 0.02] = np.nan
    sim = big[:, 3:3 + C]
    d = _cuda(big)[:, 3:3 + C]
    assert d.stride(0) == C + 9
    hq = np.sort(rng.standard_normal((nq, C)) * 8, axis=0).astype(np.float32)
    af = rng.standard_normal((nq, C)).astype(np.float32)
    af[3, 5] = np.nan
    sc = (rng.standard_normal(C) * 0.5).astype(np.float32)
    for interp in ("nearest", "linear"):
        for deg in (0, 1, 2):
            scen, coef = device.dqm_adjust(d, _cuda(af), _cuda(hq), _cuda(sc), 0, INTERP[interp], deg, want_coef=True)
            exp = D.dqm_adjust(sim, af, hq, sc, "+", interp, detrend=deg, coef=_np(coef))
            np.testing.assert_array_equal(_np(scen), exp, err_msg=f"T={T} {interp} deg={deg}")
    for deg in (0, 1, 2):
        out = _np(device.detrend(d, deg))
        coef = _np(device.poly_fit(d, deg))
        np.testing.assert_array_equal(out, sim.astype(np.float64) - D.trend_from_coef(coef, T))
        np.testing.assert_allclose(out, D.detrend(sim, deg), rtol=0, atol=1e-8 * np.nanmax(np.abs(sim)),
                                   equal_nan=True)
    fld = make_field(sim, "1990-01-01", units="K")
    g = generic.detrend(fld, deg=1)
    assert g.values.dtype == np.float64 and g.attrs == {"units": "K"} and g.dims == fld.dims
    np.testing.assert_array_equal(g.values, _np(device.detrend(_cuda(sim), 1)))


def test_dqm_headline_sample(cuda):
    """The headline series (10950 days of synthetic tasmax, 1440 cells per lat row) on a lat sub-tile sized from the
    free device memory; 2048 sampled cells and the last 128 against the oracle fed the kernel's coefficients."""
    import torch
    from xclim_b200 import device
    T, X = 10950, 1440
    free = torch.cuda.mem_get_info()[0]
    rows = int(max(4, min(180, free * 0.4 // (X * T * 14))))
    C = rows * X
    ref = device.synth(T, C, kind=1, seed=3, cells_per_lat=X, n_lat_global=rows)
    hist = device.synth(T, C, kind=1, seed=5, cells_per_lat=X, n_lat_global=rows)
    af, hq, sc = device.dqm_train(ref, hist, 20, 0)
    rng = np.random.default_rng(77)
    cells = np.unique(np.concatenate([rng.choice(C - 128, 2048, replace=False), np.arange(C - 128, C)]))
    idx = torch.from_numpy(cells).cuda()
    e_af, e_hq, e_sc = D.dqm_train(_np(ref[:, idx]), _np(hist[:, idx]), 20, "+")
    np.testing.assert_array_equal(_np(af[:, idx]), e_af)
    np.testing.assert_array_equal(_np(hq[:, idx]), e_hq)
    np.testing.assert_array_equal(_np(sc[idx]), e_sc)
    del ref
    sim = hist
    scen, coef = device.dqm_adjust(sim, af, hq, sc, 0, 1, 1, want_coef=True)
    exp = D.dqm_adjust(_np(sim[:, idx]), _np(af[:, idx]), _np(hq[:, idx]), _np(sc[idx]), "+", "linear", detrend=1,
                       coef=_np(coef[:, idx]))
    np.testing.assert_array_equal(_np(scen[:, idx]), exp)
