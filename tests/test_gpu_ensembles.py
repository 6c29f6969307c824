"""Ensemble kernels on the GPU against oracle/ensemble_oracle.py: percentiles bit for bit on both sort paths,
moments, robustness fractions and p-values, and one end-to-end run on device-resident Fields."""
import numpy as np
import pytest
import torch

from oracle import ensemble_oracle as E
from xclim_b200 import Field, TimeAxis, device, ensembles, indices, set_options

pytestmark = pytest.mark.gpu

METHODS = list(E.QUANTILE_PARAMS)
PERS = [0, 1, 10, 50, 90, 99, 100]
RS = list(range(1, 41)) + [63, 64, 65, 100, 128]


def _hostile(R, N, seed):
    """Columns with 0..R valid members, ties, +-0, +-inf and +-3.4e38."""
    rng = np.random.default_rng(seed)
    x = rng.normal(0, 10, (R, N)).astype(np.float32)
    x[:, 1::7] = np.round(x[:, 1::7])                             # ties
    nvalid = rng.integers(0, R + 1, N)
    for c in range(N):
        x[rng.permutation(R)[:R - nvalid[c]], c] = np.nan
    pool = np.array([0.0, -0.0, np.inf, -np.inf, 3.4e38, -3.4e38], np.float32)
    hit = rng.random((R, N)) < 0.08
    x[hit] = rng.choice(pool, hit.sum())
    x[:, 0] = np.nan
    if R > 1:
        x[:, 2] = np.inf
        x[0, 3], x[1:, 3] = -np.inf, 3.4e38
    return x


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def assert_bits_equal(got, exp, msg=""):
    """Same NaN positions and, elsewhere, the same bit patterns (the sign of zero included)."""
    got, exp = np.asarray(got), np.asarray(exp)
    assert got.dtype == exp.dtype, msg
    nan = np.isnan(exp)
    np.testing.assert_array_equal(np.isnan(got), nan, err_msg=msg)
    u = np.uint64 if got.dtype == np.float64 else np.uint32
    np.testing.assert_array_equal(got.view(u)[~nan], exp.view(u)[~nan], err_msg=msg)


@pytest.mark.parametrize("R", RS)
def test_percentiles_bit_exact(R):
    N = 300
    x = _hostile(R, N, R)
    xd = _dev(x)
    for method in METHODS:
        a, b = E.QUANTILE_PARAMS[method]
        got = device.ens_percentiles(xd, PERS, a, b, 1).cpu().numpy()
        exp = E.percentiles(x, PERS, a, b, 1)
        assert got.dtype == (np.float32 if R == 1 else np.float64)
        assert_bits_equal(got, exp, f"R={R} {method}")


@pytest.mark.parametrize("R", [1, 5, 32, 33, 64, 65])
@pytest.mark.parametrize("N", [1, 63, 64, 65, 127, 128, 129, 1000])
def test_percentiles_layouts_and_min_members(R, N):
    """N around whole CTAs (64 and 128 lanes), a column view of a wider buffer, min_members at its edges."""
    x = _hostile(R, N + 13, 1000 + R)
    wide = _dev(x)
    view = wide[:, 5:5 + N]
    assert view.stride(0) == N + 13
    for mm in (0, 1, R - 1, R, R + 1):
        got = device.ens_percentiles(view, [10, 50, 90], 1.0, 1.0, mm).cpu().numpy()
        assert_bits_equal(got, E.percentiles(x[:, 5:5 + N], [10, 50, 90], 1.0, 1.0, mm), f"min_members={mm}")


@pytest.mark.parametrize("R", [1, 2, 7, 30, 33, 100])
def test_moments(R):
    rng = np.random.default_rng(R)
    N = 777
    x = rng.normal(280, 8, (R, N)).astype(np.float32)
    x[rng.random((R, N)) < 0.2] = np.nan
    x[:, 0] = np.nan
    xd = _dev(x)
    mean, std, vmin, vmax = (t.cpu().numpy() for t in device.ens_moments(xd, None, 1))
    em, es, emin, emax = E.moments(x, None, 1)
    np.testing.assert_array_equal(vmin, emin)
    np.testing.assert_array_equal(vmax, emax)
    np.testing.assert_array_equal(mean, em)
    np.testing.assert_array_equal(std, es)
    # numpy in float32 (xarray's unweighted path): within R float32 ulp of the mean's magnitude
    ok = ~np.isnan(em)
    xm, xs = np.nanmean(x[:, ok], 0), np.nanstd(x[:, ok], 0)
    ulp = np.spacing(np.abs(xm)).astype(np.float64)
    assert np.all(np.abs(mean[ok] - xm) <= R * ulp)
    assert np.all(np.abs(std[ok] - xs) <= R * ulp)
    w = rng.random(R) * 3
    w[0] = 0.0
    wm, ws, wmin, wmax = (t.cpu().numpy() for t in device.ens_moments(xd, _dev(w), 2))
    rm, rs, rmin, rmax = E.moments(x, w, 2)
    assert wm.dtype == np.float64
    np.testing.assert_allclose(wm, rm, rtol=1e-12)
    np.testing.assert_allclose(ws, rs, rtol=1e-12, atol=1e-300)
    np.testing.assert_array_equal(wmin, rmin)


def _series(R, T, C, seed):
    rng = np.random.default_rng(seed)
    x = (rng.normal(0, 1, (R, T, C)) + rng.normal(0, 0.5, (R, 1, C))).astype(np.float32)
    x[0, 3, ::5] = np.nan              # partial NaN: invalid member
    x[R - 1, :, 1::9] = np.nan         # a full NaN series
    return x


TESTS = [(None, {}), ("threshold", {"abs_thresh": 0.3}), ("threshold", {"rel_thresh": 0.5}),
         ("ttest", {"p_change": 0.05}), ("welch-ttest", {"p_change": 0.1})]


@pytest.mark.parametrize("test, kw", TESTS)
@pytest.mark.parametrize("strict", [True, False])
@pytest.mark.parametrize("weighted", [False, True])
def test_robustness_against_oracle(test, kw, strict, weighted):
    R, C = 9, 517
    fut, ref = _series(R, 12, C, 1), _series(R, 17, C, 2)
    w = np.linspace(0.5, 2.0, R) if weighted else None
    f = Field(fut, ("realization", "time", "x"), None, {}, {}, "tas")
    r = Field(ref, ("realization", "time", "x"), None, {}, {}, "tas")
    out = ensembles.robustness_fractions(f, r, test=test, weights=w, strict_sign=strict, **kw)
    code = {"abs_thresh": "abs_thresh", "rel_thresh": "rel_thresh"}.get(next(iter(kw), None), test)
    frac, pv = device.ens_robustness(_dev(fut), _dev(ref), None if w is None else _dev(w), _lib_code(code),
                                     next(iter(kw.values()), 0.0), strict, test in ("ttest", "welch-ttest"))
    exp, p, chg = E.robustness(fut, ref, test, w, strict, **kw)
    if pv is not None:
        pk = pv.cpu().numpy()
        assert np.array_equal(np.isnan(pk), np.isnan(p))
        ok = ~np.isnan(p)
        # the kernel's float64 p rounded once to float32, against the float64 oracle
        np.testing.assert_allclose(pk[ok], p[ok].astype(np.float32), rtol=1e-6, atol=1e-30)
        np.testing.assert_array_equal(out["pvals"].values, pk)
    for k, name in enumerate(E.FRACTIONS):
        np.testing.assert_array_equal(frac[k].cpu().numpy(), exp[name], err_msg=name)
        np.testing.assert_array_equal(out[name].values, exp[name], err_msg=name)


def _lib_code(name):
    from xclim_b200 import _lib
    return _lib.ENS_TESTS[name]


def test_robustness_pvalues_float64_within_1e12():
    """The pvals output is float32; the float64 p-values behind `changed` are checked through p_change set just
    above and below each oracle p-value."""
    R, C = 4, 256
    fut, ref = _series(R, 10, C, 7), _series(R, 14, C, 8)
    _, p, _ = E.robustness(fut, ref, "welch-ttest")
    for r in range(R):
        for c in range(0, C, 37):
            if np.isnan(p[r, c]):
                continue
            one = lambda a: _dev(a[r:r + 1, :, c:c + 1])  # noqa: E731
            hi, _ = device.ens_robustness(one(fut), one(ref), None, _lib_code("welch-ttest"), p[r, c] * (1 + 1e-12),
                                          True, False)
            lo, _ = device.ens_robustness(one(fut), one(ref), None, _lib_code("welch-ttest"), p[r, c] * (1 - 1e-12),
                                          True, False)
            valid = float(hi[5].item()) > 0
            if valid:
                assert hi[0].item() == 1.0 and lo[0].item() == 0.0, (r, c)


def test_robustness_known_answers_end_to_end():
    # tests/test_ensembles.py:685-720
    d = Field(torch.tensor([-2, 1, -2, -1, 0, 0], dtype=torch.float32).cuda(), ("realization",), None, {}, {}, "d")
    fr = ensembles.robustness_fractions(d, test="threshold", abs_thresh=1.5)
    assert [float(fr[k].values) for k in ("changed", "changed_positive", "positive", "agree")] == \
        [2 / 6, 0.0, 1 / 6, 3 / 6]
    d = Field(np.array([-2, 1, -2, -1], np.float32), ("realization",), None, {}, {}, "d")
    fr = ensembles.robustness_fractions(d, test="threshold", abs_thresh=1.5, weights=np.array([4, 3, 2, 1]))
    assert [float(fr[k].values) for k in ("changed", "positive", "agree")] == [0.6, 0.3, 0.7]
    d = Field(np.array([-2, 1, -2, -1, 2, 0], np.float32), ("realization",), None, {}, {}, "d")
    fr = ensembles.robustness_fractions(d, test=None, strict_sign=False)
    assert [float(fr[k].values) for k in ("changed", "positive", "agree")] == [1, 3 / 6, 4 / 6]
    nan = Field(np.full((20, 10), np.nan, np.float32), ("realization", "time"), None, {}, {}, "tas")
    fr = ensembles.robustness_fractions(nan, nan, test="ttest")
    assert float(fr["changed"].values) == 0 and float(fr["valid"].values) == 0


def test_end_to_end_tg_mean_ensemble_on_device():
    R, Y, X = 6, 4, 40
    ta = TimeAxis.daily("2000-01-01", 365 * 6, "noleap")
    members = []
    for r in range(R):
        tas = device.synth(365 * 6, Y * X, kind=1, seed=10 + r, cells_per_lat=X, n_lat_global=Y)
        members.append(Field(tas.reshape(-1, Y, X), ("time", "lat", "lon"), ta, {}, {"units": "K"}, "tas"))
    with set_options(device_outputs=True):
        tg = [indices.tg_mean(m, freq="YS") for m in members]
        assert all(t.values.is_cuda for t in tg)
        ens = ensembles.create_ensemble(tg)
        assert ens.values.is_cuda and ens.dims == ("realization", "time", "lat", "lon")
        pct = ensembles.ensemble_percentiles(ens, values=[10, 50, 90])
        fut = Field(ens.values[:, 3:], ens.dims, None, {}, {}, "tg_mean")
        ref = Field(ens.values[:, :3], ens.dims, None, {}, {}, "tg_mean")
        fr = ensembles.robustness_fractions(fut, ref, test="ttest")
    assert list(pct) == [f"{ens.name}_p{p}" for p in (10, 50, 90)]
    assert pct[f"{ens.name}_p50"].values.is_cuda and fr["agree"].values.is_cuda
    host = ens.values.cpu().numpy()
    exp = E.percentiles(host, [10, 50, 90])
    for k, p in enumerate((10, 50, 90)):
        assert_bits_equal(pct[f"{ens.name}_p{p:02d}"].values.cpu().numpy(), exp[k])
    efr, _, _ = E.robustness(host[:, 3:], host[:, :3], "ttest", None, True)
    np.testing.assert_array_equal(fr["positive"].values.cpu().numpy(), efr["positive"])
    np.testing.assert_array_equal(fr["valid"].values.cpu().numpy(), efr["valid"])


def test_percentiles_zero_maximum_keeps_the_reference_sign():
    """_nan_quantile clamps a top percentile to index -1: max - 0 * (1 - g), which turns a -0 maximum into +0 when
    no member is NaN, and keeps -0 (the NaN-fallback maximum) when one is."""
    x = np.array([[-0.0, -0.0, -1.0], [-1.0, -0.0, np.nan], [-2.0, -3.0, -0.0]], np.float32)
    got = device.ens_percentiles(_dev(x), [100, 50, 0], 1.0, 1.0, 1).cpu().numpy()
    assert_bits_equal(got, E.percentiles(x, [100, 50, 0]))
    assert np.signbit(got[0]).tolist() == [False, False, True]


@pytest.mark.parametrize("calendar", ["noleap", "standard"])
@pytest.mark.parametrize("weighted", [False, True])
def test_robustness_ipcc_ar6_c(calendar, weighted):
    """ipcc-ar6-c: |delta| > sqrt(2/20) 1.645 sigma, sigma the std of the YS means of ref about their least-squares
    line on the actual YS timestamps (leap years in the standard calendar), against numpy.polyfit."""
    R, C, ny = 7, 389, 12
    days = sum(366 if (calendar == "standard" and y % 4 == 0) else 365 for y in range(1995, 1995 + ny))
    ta_ref = TimeAxis.daily("1995-01-01", days, calendar)
    rng = np.random.default_rng(3)
    trend = np.linspace(0, 1.5, days, dtype=np.float32)[None, :, None]
    ref = (rng.normal(0, 1, (R, days, C)) + trend + rng.normal(0, 0.3, (R, 1, C))).astype(np.float32)
    ref[1, 40, ::3] = np.nan                       # invalid members in some cells
    fut = (rng.normal(0.25, 1, (R, 400, C))).astype(np.float32)
    w = np.linspace(2.0, 0.5, R) if weighted else None
    f = Field(fut, ("realization", "time", "x"), None, {}, {}, "tas")
    r = Field(ref, ("realization", "time", "x"), ta_ref, {}, {}, "tas")
    out = ensembles.robustness_fractions(f, r, test="ipcc-ar6-c", weights=w)
    assert "pvals" not in out and out["changed"].attrs["test"] == "ipcc-ar6-c"
    poff = ta_ref.period_offsets("YS")
    starts = np.array([np.datetime64(f"{y}-01-01") for y in range(1995, 1995 + ny)])
    ys = (starts - starts[0]).astype("timedelta64[D]").astype(np.float64)
    if calendar == "noleap":
        ys = 365.0 * np.arange(ny)
    exp, _, chg = E.robustness(fut, ref, "ipcc-ar6-c", w, True, poff=poff, ys_time=ys)
    assert 0 < chg.mean() < 1
    for name in E.FRACTIONS:
        np.testing.assert_array_equal(out[name].values, exp[name], err_msg=name)
    with pytest.raises(NotImplementedError, match="ref_pi"):
        ensembles.robustness_fractions(f, r, test="ipcc-ar6-c", ref_pi=r)
