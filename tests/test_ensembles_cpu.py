"""Ensemble statistics without a GPU: the host build of the Student-t distribution against scipy, the oracle
against the reference tests' known answers and scipy's tests, and the host layer of xclim_b200.ensembles over
the oracle-backed stand-ins (tests/fake_ensemble.py)."""
import os
import sys
import warnings

import numpy as np
import pytest
import scipy.special as sps
import scipy.stats as st
import torch
from scipy.stats.mstats import mquantiles

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ensemble_host_build as H  # noqa: E402
import fake_ensemble  # noqa: E402
import mini_xarray as mx  # noqa: E402
from oracle import ensemble_oracle as E  # noqa: E402
from xclim_b200 import Field, TimeAxis, ensembles, set_options  # noqa: E402

DFS_SMALL = list(range(1, 31)) + [0.5, 1.5, 2.7, 7.3, 33.3, 50, 99.5, 100, 250.25, 1000, 1234.5, 2000, 5000]
DFS_LARGE = [9999.9, 1e4]
TS = [1e200, 1e20, 1e6, 300, 100, 40, 20, 10, 5, 3, 2, 1.5, 1, 0.5, 0.1, 0.01]


# ---------------------------------------------------------------------------------------- Student t
@pytest.mark.parametrize("dfs, tol", [(DFS_SMALL, 1e-13), (DFS_LARGE, 1e-12)])
def test_stdtr_host_build_matches_scipy(dfs, tol):
    """Both tails, integer and non-integer df.  Above df = 5000, near the centre of the distribution, the
    continued fraction runs for thousands of terms and its rounding reaches ~6e-13: the tolerance there is 1e-12."""
    D, T = np.meshgrid(np.asarray(dfs, float), np.asarray(TS + [-t for t in TS]), indexing="ij")
    ref = sps.stdtr(D, T)
    got = H.stdtr(D, T)
    keep = ref > 1e-290     # subnormal results carry no relative precision (scipy gives 0 at t = -1e200)
    np.testing.assert_allclose(got[keep], ref[keep], rtol=tol, atol=0)
    assert np.all(got[~keep] < 1e-100)      # the true tails there: 3.2e-101 (df = 0.5), 3.2e-201 (df = 1)


def test_stdtr_near_zero_against_closed_forms():
    """Close to t = 0 scipy's stdtr forms 1 - I_x and loses ~|log10 t| digits; the Cauchy (df = 1) and df = 2
    closed forms are exact references there."""
    t = np.array([-1e-8, -1e-5, -1e-3, 1e-3, 1e-5, 1e-8, 1e-300, -1e-300])
    np.testing.assert_allclose(H.stdtr(1.0, t), 0.5 + np.arctan(t) / np.pi, rtol=1e-15)
    np.testing.assert_allclose(H.stdtr(2.0, t), 0.5 + t / (2 * np.sqrt(2 + t * t)), rtol=1e-15)


def test_stdtr_edges():
    out = H.stdtr([1.0, 1.0, 3.0, 3.0, 0.0, -1.0, np.nan, 2.0], [0.0, np.inf, -np.inf, np.nan, 1.0, 1.0, 1.0, -0.0])
    np.testing.assert_array_equal(out[:3], [0.5, 1.0, 0.0])
    assert np.isnan(out[3:7]).all()
    assert out[7] == 0.5


def test_host_ttests_match_scipy_in_float64():
    rng = np.random.default_rng(1)
    for n1, n2 in [(2, 2), (3, 7), (30, 30), (200, 17)]:
        f = rng.normal(0.3, 1.0, n1)
        r = rng.normal(0.0, 2.0, n2)
        m1, m2 = f.mean(), r.mean()
        p1 = H.ttest_1samp_p(n1, m1, ((f - m1) ** 2).sum(), m2)
        assert p1 == pytest.approx(st.ttest_1samp(f, m2)[1], rel=1e-11)
        p2 = H.welch_ttest_p(n1, m1, ((f - m1) ** 2).sum(), n2, m2, ((r - m2) ** 2).sum())
        assert p2 == pytest.approx(st.ttest_ind(f, r, equal_var=False)[1], rel=1e-11)
    assert np.isnan(H.ttest_1samp_p(1, 1.0, 0.0, 0.0))
    assert H.welch_ttest_p(3, 1.0, 0.0, 3, 2.0, 0.0) == 0.0          # zero variances: t = -inf, df set to 1
    assert np.isnan(H.welch_ttest_p(3, 1.0, 0.0, 3, 1.0, 0.0))


# ---------------------------------------------------------------------------------------- oracle
def test_oracle_known_answers_deltas():
    # tests/test_ensembles.py:685-707
    fr, p, _ = E.robustness(np.array([-2, 1, -2, -1, 0, 0], np.float32), test="threshold", abs_thresh=1.5)
    assert (fr["changed"], fr["changed_positive"], fr["positive"], fr["agree"]) == (2 / 6, 0.0, 1 / 6, 3 / 6)
    fr, _, _ = E.robustness(np.array([-2, 1, -2, -1], np.float32), test="threshold", abs_thresh=1.5,
                            weights=[4, 3, 2, 1])
    assert (fr["changed"], fr["positive"], fr["agree"]) == (0.6, 0.3, 0.7)
    fr, _, _ = E.robustness(np.array([-2, 1, -2, -1, 2, 0], np.float32), strict_sign=False)
    assert (fr["changed"], fr["positive"], fr["agree"]) == (1, 3 / 6, 4 / 6)


def test_oracle_known_answers_all_nan():
    # tests/test_ensembles.py:709-720
    nan = np.full((20, 10), np.nan, np.float32)
    fr, p, _ = E.robustness(nan, nan, test="ttest")
    assert fr["changed"] == 0 and fr["valid"] == 0
    assert np.isnan(p).all()


@pytest.mark.parametrize("method", list(E.QUANTILE_PARAMS))
def test_oracle_percentiles_match_mquantiles(method):
    # tests/test_ensembles.py:120-215: scipy's mquantiles with the same plotting positions, NaN members masked
    rng = np.random.default_rng(5)
    x = rng.normal(280, 5, (11, 40)).astype(np.float32)
    x[2, 7] = x[5, 7] = np.nan
    a, b = E.QUANTILE_PARAMS[method]
    got = E.percentiles(x, [10, 50, 90], a, b)
    for c in (0, 7, 39):
        exp = mquantiles(np.ma.fix_invalid(x[:, c]), [0.1, 0.5, 0.9], alphap=a, betap=b)
        np.testing.assert_allclose(got[:, c], exp, rtol=1e-6)
    assert got.dtype == np.float64
    assert E.percentiles(x[:1], [50]).dtype == np.float32


def _scipy_wrappers(f, r, test):
    """ensembles/_robustness.py:529-534 and :562-565 on one member, float32 as there"""
    if np.isnan(f).all() or np.isnan(r).all():
        return np.nan
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if test == "ttest":
            return st.ttest_1samp(f, np.nanmean(r)[..., None], axis=-1, nan_policy="omit")[1]
        return st.ttest_ind(f, r, axis=-1, equal_var=False, nan_policy="omit")[1]


@pytest.mark.parametrize("test", ["ttest", "welch-ttest"])
def test_oracle_pvalues_match_scipy_tests(test):
    """The float64 oracle against scipy's float32 tests: p-values within float32 rounding, `changed` equal except
    where scipy's p lies within that tolerance of p_change."""
    rng = np.random.default_rng(9)
    R, C = 12, 64
    fut = rng.normal(0.2, 1.0, (R, 15, C)).astype(np.float32)
    ref = rng.normal(0.0, 1.0, (R, 20, C)).astype(np.float32)
    fut[0, 3, :5] = np.nan
    ref[1, :, 7] = np.nan
    _, p, chg = E.robustness(fut, ref, test)
    sp = np.array([[_scipy_wrappers(fut[r, :, c], ref[r, :, c], test) for c in range(C)] for r in range(R)])
    both = np.isnan(sp) == np.isnan(p)
    assert both.all()
    ok = ~np.isnan(sp)
    np.testing.assert_allclose(p[ok], sp[ok], rtol=2e-5, atol=1e-7)
    near = np.abs(sp - 0.05) <= 2e-5 * 0.05 + 1e-7
    assert np.all((chg == (sp < 0.05)) | near)


# ---------------------------------------------------------------------------------------- host layer
@pytest.fixture
def fake(monkeypatch):
    return fake_ensemble.install(monkeypatch)


def _ens_field(R=5, T=4, Y=3, X=6, seed=0, name="tg_mean"):
    rng = np.random.default_rng(seed)
    v = rng.normal(280, 3, (R, T, Y, X)).astype(np.float32)
    v[1, 0, 0, 0] = np.nan
    ta = TimeAxis.daily("2000-01-01", T, "noleap")
    return Field(v, ("realization", "time", "lat", "lon"), ta, {"lat": np.arange(Y)}, {"units": "K",
                 "description": "Mean temperature"}, name)


def test_percentiles_field_split_and_dtypes(fake):
    ens = _ens_field()
    out = ensembles.ensemble_percentiles(ens)
    assert list(out) == ["tg_mean_p10", "tg_mean_p50", "tg_mean_p90"]
    p50 = out["tg_mean_p50"]
    assert p50.dims == ("time", "lat", "lon") and p50.values.dtype == np.float64
    assert p50.attrs["description"] == "Mean temperature 50th percentile of ensemble."
    np.testing.assert_array_equal(p50.values, E.percentiles(ens.values, [50])[0])
    one = ensembles.ensemble_percentiles(Field(ens.values[:1], ens.dims, ens.time, {}, {}, "x"), values=[50])
    assert one["x_p50"].values.dtype == np.float32
    np.testing.assert_array_equal(one["x_p50"].values, ens.values[0])


def test_percentiles_no_split_transposed_and_min_members(fake):
    ens = _ens_field()
    out = ensembles.ensemble_percentiles(ens, values=[25, 75], split=False, method="hazen")
    assert out.dims == ("time", "lat", "lon", "percentiles")
    np.testing.assert_array_equal(out.coords["percentiles"], [25, 75])
    exp = np.moveaxis(E.percentiles(ens.values, [25, 75], 0.5, 0.5), 0, -1)
    np.testing.assert_array_equal(out.values, exp)
    tr = Field(np.ascontiguousarray(np.transpose(ens.values, (3, 2, 1, 0))), ("lon", "lat", "time", "realization"),
               ens.time, {}, {}, "tg_mean")
    out_t = ensembles.ensemble_percentiles(tr, values=[25, 75], split=False, method="hazen")
    assert out_t.dims == ("lon", "lat", "time", "percentiles")
    np.testing.assert_array_equal(out_t.values, np.transpose(exp, (2, 1, 0, 3)))
    full = ensembles.ensemble_percentiles(ens, min_members=None)
    assert np.isnan(full["tg_mean_p50"].values[0, 0, 0])
    assert np.isfinite(full["tg_mean_p50"].values[1]).all()


def test_mean_std_max_min_field_and_weights(fake):
    ens = _ens_field()
    out = ensembles.ensemble_mean_std_max_min(ens)
    assert list(out) == ["tg_mean_mean", "tg_mean_stdev", "tg_mean_max", "tg_mean_min"]
    assert all(v.values.dtype == np.float32 for v in out.values())
    assert out["tg_mean_mean"].attrs["description"] == "Mean temperature : mean_mean of ensemble"    # _base.py:205
    np.testing.assert_allclose(out["tg_mean_mean"].values, np.nanmean(ens.values, 0), rtol=1e-6)
    np.testing.assert_allclose(out["tg_mean_stdev"].values, np.nanstd(ens.values, 0), rtol=1e-4)
    np.testing.assert_array_equal(out["tg_mean_max"].values, np.nanmax(ens.values, 0))
    w = ensembles.ensemble_mean_std_max_min(ens, weights=np.array([1, 0.1, 3.5, 5, 0.0]))
    assert w["tg_mean_mean"].values.dtype == np.float64 and w["tg_mean_max"].values.dtype == np.float32
    with pytest.raises(ValueError, match="cannot contain missing values"):
        ensembles.ensemble_mean_std_max_min(ens, weights=np.array([1, np.nan, 1, 1, 1]))


def test_column_walk_with_tiny_slabs(fake):
    ens = _ens_field(R=7, T=3, Y=4, X=9)
    exp = ensembles.ensemble_percentiles(ens, split=False)
    exp_m = ensembles.ensemble_mean_std_max_min(ens)
    with set_options(stream_min_bytes=0, stream_slab_bytes=7 * 4 * 10):
        got = ensembles.ensemble_percentiles(ens, split=False)
        got_m = ensembles.ensemble_mean_std_max_min(ens)
    np.testing.assert_array_equal(got.values, exp.values)
    for k in exp_m:
        np.testing.assert_array_equal(got_m[k].values, exp_m[k].values)
    N = 3 * 4 * 9
    widths = [b[0] // 4 for b in fake.boxes]
    assert widths[:N // 10 + 1] == [10] * (N // 10) + [N % 10] and all(b[1] == 7 for b in fake.boxes)


def test_mini_xarray_boundary(fake, monkeypatch):
    mx.install(monkeypatch)
    ens = _ens_field()
    da = mx.DataArray(ens.values, dims=ens.dims, coords={"lat": np.arange(3)}, attrs={"units": "K"}, name="tg")
    out = ensembles.ensemble_percentiles(da, values=[50])
    p = out["tg_p50"]
    assert isinstance(p, mx.DataArray) and p.dims == ("time", "lat", "lon") and p.values.dtype == np.float64
    fr = ensembles.robustness_fractions(da, da, test="ttest")
    assert isinstance(fr["changed"], mx.DataArray) and fr["pvals"].dims == ("realization", "lat", "lon")
    assert fr["pvals"].values.dtype == np.float32 and fr["changed"].values.dtype == np.float64


def test_dict_of_variables_is_reduced_variable_by_variable(fake):
    a, b = _ens_field(name="a"), _ens_field(seed=3, name="b")
    out = ensembles.ensemble_percentiles({"a": a, "b": b}, values=[10])
    assert list(out) == ["a_p10", "b_p10"]
    m = ensembles.ensemble_mean_std_max_min({"a": a, "b": b})
    assert list(m) == ["a_mean", "a_stdev", "a_max", "a_min", "b_mean", "b_stdev", "b_max", "b_min"]


def test_create_ensemble(fake):
    m = [Field(np.full((4, 2), float(k), np.float32), ("time", "x"), None, {}, {"units": "K"}, "v") for k in range(3)]
    ens = ensembles.create_ensemble(m)
    assert ens.dims == ("realization", "time", "x") and ens.shape == (3, 4, 2)
    np.testing.assert_array_equal(ens.coords["realization"], [0, 1, 2])
    ens = ensembles.create_ensemble({"a": m[0], "b": m[1]})
    np.testing.assert_array_equal(ens.coords["realization"], ["a", "b"])
    for kw in ({"resample_freq": "MS"}, {"calendar": "noleap"}, {"multifile": True}, {"cal_kwargs": {"x": 1}}):
        with pytest.raises(NotImplementedError):
            ensembles.create_ensemble(m, **kw)
    with pytest.raises(NotImplementedError, match="glob"):
        ensembles.create_ensemble("/data/*.nc")
    with pytest.raises(NotImplementedError, match="glob"):
        ensembles.create_ensemble(["a.nc", "b.nc"])
    bad = Field(np.zeros((5, 2), np.float32), ("time", "x"), None, {}, {}, "v")
    with pytest.raises(NotImplementedError, match="aligning"):
        ensembles.create_ensemble([m[0], bad])
    with pytest.raises(ValueError):
        ensembles.create_ensemble([])


def test_errors(fake):
    ens = _ens_field()
    with pytest.raises(NotImplementedError, match="weighted"):
        ensembles.ensemble_percentiles(ens, weights=np.ones(5))
    with pytest.raises(ValueError, match="method"):
        ensembles.ensemble_percentiles(ens, method="nearest")
    d = Field(np.array([-2, 1, -2, -1], np.float32), ("realization",), None, {}, {}, "d")
    with pytest.raises(ValueError, match="When deltas are given"):
        ensembles.robustness_fractions(d, test="ttest")
    with pytest.raises(ValueError, match="One and only one"):
        ensembles.robustness_fractions(d, test="threshold")
    with pytest.raises(ValueError, match="One and only one"):
        ensembles.robustness_fractions(d, test="threshold", abs_thresh=1, rel_thresh=1)
    with pytest.raises(ValueError, match="must be one of"):
        ensembles.robustness_fractions(ens, ens, test="nope")
    for t in ("mannwhitney-utest", "brownforsythe-test"):
        with pytest.raises(NotImplementedError):
            ensembles.robustness_fractions(ens, ens, test=t)
    with pytest.raises(NotImplementedError, match="ref_pi"):
        ensembles.robustness_fractions(ens, ens, test="ipcc-ar6-c", ref_pi=ens)
    with pytest.raises(ValueError, match="time"):
        ensembles.robustness_fractions(ens, test="threshold", abs_thresh=1.0)

    class AtLeastNValid:
        pass

    with pytest.raises(NotImplementedError, match="MissingAny"):
        ensembles.robustness_fractions(ens, ens, test="ttest", invalid=AtLeastNValid())

    class MissingAny:
        pass

    ensembles.robustness_fractions(ens, ens, test="ttest", invalid=MissingAny())


def test_robustness_known_answers_through_host_layer(fake):
    d = Field(np.array([-2, 1, -2, -1, 0, 0], np.float32), ("realization",), None, {}, {}, "d")
    fr = ensembles.robustness_fractions(d, test="threshold", abs_thresh=1.5)
    assert [float(fr[k].values) for k in ("changed", "changed_positive", "positive", "agree")] == \
        [2 / 6, 0.0, 1 / 6, 3 / 6]
    assert fr["changed"].attrs["test"] == "threshold" and "pvals" not in fr
    d = Field(np.array([-2, 1, -2, -1], np.float32), ("realization",), None, {}, {}, "d")
    fr = ensembles.robustness_fractions(d, test="threshold", abs_thresh=1.5, weights=np.array([4, 3, 2, 1]))
    assert [float(fr[k].values) for k in ("changed", "positive", "agree")] == [0.6, 0.3, 0.7]
    nan = Field(np.full((20, 10), np.nan, np.float32), ("realization", "time"), None, {}, {}, "tas")
    fr = ensembles.robustness_fractions(nan, nan, test="ttest")
    assert float(fr["changed"].values) == 0 and float(fr["valid"].values) == 0
    assert fr["pvals"].dims == ("realization",) and np.isnan(fr["pvals"].values).all()


def test_robustness_categories():
    # tests/test_ensembles.py:730-739
    changed = np.array([0.5, 0.8, 1, 1])
    agree = np.array([1, 0.5, 0.5, 1])
    np.testing.assert_array_equal(ensembles.robustness_categories(changed, agree), [2, 3, 3, 1])
    t = ensembles.robustness_categories(torch.tensor(changed), torch.tensor(agree), valid=torch.tensor([1, 1, 0, 1.]))
    assert isinstance(t, torch.Tensor) and t.tolist() == [2, 3, 99, 1]
    f = ensembles.robustness_categories({"changed": Field(changed, ("lat",), None, {"lat": np.arange(4)}, {}, "c"),
                                         "agree": agree, "valid": np.ones(4)})
    assert f.attrs["flag_values"] == [1, 2, 3]
    assert f.attrs["flag_meanings"] == "robust_signal no_change_or_no_signal conflicting_signal"
    np.testing.assert_array_equal(f.values, [2, 3, 3, 1])


def test_total_order_oracle_equals_nan_quantile():
    """The ensemble oracle's percentiles are xclim_oracle.nan_quantile (pinned to the reference by
    tests/golden/ref_quantile.npz) value for value; only the sign of a zero result is fixed."""
    from oracle import xclim_oracle as O
    rng = np.random.default_rng(4)
    for R in (2, 3, 7, 30, 65):
        x = rng.normal(0, 3, (R, 400)).astype(np.float32)
        x[rng.random(x.shape) < 0.2] = np.nan
        pool = np.array([0.0, -0.0, np.inf, -np.inf, 3.4e38, -3.4e38], np.float32)
        hit = rng.random(x.shape) < 0.15
        x[hit] = rng.choice(pool, hit.sum())
        for a, b in E.QUANTILE_PARAMS.values():
            per = [0, 1, 10, 50, 90, 99, 100]
            np.testing.assert_array_equal(E.percentiles(x, per, a, b), O.nan_quantile(x, np.array(per) / 100, a, b))


def test_ipcc_gamma_oracle_known_answer():
    """Residuals of a line are +-e about it, whatever the abscissa's origin and unit: sigma = e."""
    x = np.array([0, 365, 731, 1096, 1461, 1827], float)      # YS timestamps in days, leap years included
    y = 2.0 + 1e-3 * x + 0.25 * np.array([1, -1, 1, -1, 1, -1])
    got = E.ipcc_ar6_c_gamma(y[None, :, None], x)
    res = y - np.polyval(np.polyfit(x, y, 1), x)
    assert got[0, 0] == pytest.approx(np.sqrt(2 / 20) * 1.645 * np.sqrt(np.mean(res ** 2)), rel=1e-12)
    assert E.ipcc_ar6_c_gamma(np.array([[[np.nan]] * 6]).reshape(1, 6, 1), x)[0, 0] != 0    # all NaN: NaN


def test_ipcc_and_pvals_dims_through_host_layer(fake):
    R, T, X = 4, 365 * 5, 3
    rng = np.random.default_rng(2)
    ta = TimeAxis.daily("2001-01-01", T, "standard")
    ref = Field(rng.normal(0, 1, (T, R, X)).astype(np.float32), ("time", "realization", "x"), ta, {}, {}, "tas")
    fut = Field(rng.normal(1, 1, (X, T, R)).astype(np.float32), ("x", "time", "realization"), None, {}, {}, "tas")
    fr = ensembles.robustness_fractions(fut, ref, test="ipcc-ar6-c")
    assert fr["changed"].dims == ("x",) and "pvals" not in fr
    assert "ref_pi=None" in fr["changed"].attrs["description"]
    fr = ensembles.robustness_fractions(fut, ref, test="ttest")
    assert fr["pvals"].dims == ("x", "realization") and fr["pvals"].values.shape == (X, R)
