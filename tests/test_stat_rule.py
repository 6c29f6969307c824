"""CPU checks of the per-period float statistic rule (oracle/stat_rule.py) that tests/test_gpu_stat_rule.py holds
the kernels to bit for bit: agreement with the reference restatements (xclim_oracle, etccdi_oracle) within the
tolerances the other tests use, sums that are sequential rather than pairwise, a variance formula with every
operation rounded, and constant cells whose variance is exactly 0."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import etccdi_oracle as E
from oracle import stat_rule as R
from oracle import xclim_oracle as O

POFF = np.array([0, 1, 31, 59, 60, 181, 365, 425], np.int32)
OPS = [">", "<", ">=", "<=", "==", "!="]


def _field(seed, T=425, C=12):
    rng = np.random.default_rng(seed)
    x = (280.0 + 8.0 * rng.standard_normal((T, C))).astype(np.float32)
    x[:, :4] = np.round(rng.gamma(0.4, 6.0, (T, 4)) * 2) / 2       # quantised: ties with the thresholds
    x[rng.random(x.shape) < 0.05] = np.nan
    x[:, 5] = np.nan
    return x


def _close(got, exp, stat, msg=""):
    if stat == "count":
        np.testing.assert_array_equal(got, exp, err_msg=msg)
    else:
        np.testing.assert_allclose(got, exp, rtol=1e-5, atol=1e-4 if stat in ("std", "var") else 0, equal_nan=True,
                                   err_msg=msg)


@pytest.mark.parametrize("stat", R.STATS)
def test_period_stat_matches_reference(stat):
    x = _field(1)
    _close(R.period_stat(x, POFF, stat), O.resample_reduce(x.astype(np.float64), POFF, stat), stat)
    for op in OPS:
        y = np.where(O.compare(x, op, 1.0), x, np.nan).astype(np.float64)
        _close(R.period_stat(x, POFF, stat, "where", op, 1.0), O.resample_reduce(y, POFF, stat), stat, op)
    for op in (">", "<", ">=", "<="):
        t = 280.0 if stat != "sum" else 1.0
        d = (x - np.float32(t)) if op in (">", ">=") else (np.float32(t) - x)
        y = np.where(np.isnan(d), np.nan, np.maximum(d, 0)).astype(np.float64)
        _close(R.period_stat(x, POFF, stat, "excess", op, t), O.resample_reduce(y, POFF, stat), stat, op)
    if stat == "sum":
        np.testing.assert_allclose(R.period_stat(x, POFF, "sum", "excess", ">", 1.0),
                                   O.cumulative_difference(x, 1.0, ">", POFF), rtol=1e-5)


def test_range_stat_matches_reference():
    lo = _field(2)
    hi = (lo + np.abs(_field(3) - 280.0)).astype(np.float32)
    for stat in ("mean", "max", "min", "std", "sum", "count", "var"):
        np.testing.assert_allclose(R.range_stat(lo, hi, POFF, stat), E.daily_temperature_range(lo, hi, POFF, stat),
                                   rtol=2e-6, atol=2e-5, equal_nan=True, err_msg=stat)
    np.testing.assert_allclose(R.range_stat(lo, hi, POFF, "mean", variability=True),
                               E.daily_temperature_range_variability(lo, hi, POFF), rtol=2e-6, atol=2e-5,
                               equal_nan=True)


@pytest.mark.parametrize("before", [True, False])
@pytest.mark.parametrize("red", ["mean", "std"])
def test_run_stat_matches_reference(red, before):
    x = _field(4)
    for op in OPS:
        m = O.compare(x, op, 1.0)
        for window in (1, 2, 4):
            got = O.resample_and_rl(m, before, R.run_stat, poff=POFF, reducer=red, window=window)
            exp = O.resample_and_rl(m, before, O.rle_statistics, poff=POFF, reducer=red, window=window)
            np.testing.assert_allclose(got, exp, rtol=1e-5, atol=0, err_msg=f"{op} w={window}")
    # known answer: runs of 1, 2 and 4 steps -> mean 7/3, std sqrt(21/3 - 49/9)
    m = np.array([1, 0, 1, 1, 0, 1, 1, 1, 1], bool)[:, None]
    assert R.run_stat(m, "mean", 1)[0] == np.float32(7 / 3)
    assert R.run_stat(m, "std", 1)[0] == np.float32(np.sqrt(21 / 3 - (7 / 3) ** 2))
    assert R.run_stat(m, "std", 5)[0] == 0.0                     # no run: 0


@pytest.mark.parametrize("before", [True, False])
def test_run_maxsum_matches_reference(before):
    x = _field(5)
    for op in (">", "<", ">=", "<="):
        for thr in (1.0, 280.0):
            t32 = np.float32(thr)
            excess = np.where(np.isnan(x), 0, np.clip((x - t32) if op in (">", ">=") else (t32 - x), 0, None))
            for window in (1, 3):
                exp = O.resample_and_rl(excess.astype(np.float64), before, O.windowed_max_run_sum, window, poff=POFF)
                np.testing.assert_allclose(R.run_maxsum(x, POFF, op, thr, window, before), exp, rtol=1e-5, atol=1e-6,
                                           err_msg=f"{op} {thr} w={window}")


def test_sums_thr_matches_reference():
    rng = np.random.default_rng(6)
    x = _field(6)[:, :4]
    thr = np.where(rng.random((1, 4)) < 0.5, 1.0, 2.5 + 1e-9)
    for op in (">", ">="):
        s_thr, s_wet = R.sums_thr(x, POFF, op, thr, 1.0)
        over = np.where(O.compare(x, op, thr), x, np.float32(0))
        total = np.where(O.compare(x, op, 1.0), x, np.float32(0))
        for got, v in ((s_thr, over), (s_wet, total)):
            exp = np.stack([v[s:e].sum(axis=0, dtype=np.float64) for s, e in O._groups(POFF)]).astype(np.float32)
            np.testing.assert_allclose(got, exp, rtol=1e-6)


def _pairwise(v):
    return v[0] if len(v) == 1 else _pairwise(v[:len(v) // 2]) + _pairwise(v[len(v) // 2:])


def test_sums_are_sequential_not_pairwise():
    """2^60 + 1 rounds back to 2^60 in float64: one add at a time the total is 1, pairwise it is 0."""
    col = np.array([2.0 ** 60, 1.0, -2.0 ** 60, 1.0], np.float32)
    seq = 0.0
    for v in col.astype(np.float64).tolist():
        seq += v
    pw = _pairwise(col.astype(np.float64).tolist())
    assert (np.float32(seq), np.float32(pw)) == (1.0, 0.0)
    x, poff = col[:, None], np.array([0, 4])
    assert R.period_stat(x, poff, "sum")[0, 0] == 1.0
    assert R.period_stat(x, poff, "mean")[0, 0] == np.float32(0.25)
    assert R.range_stat(np.zeros_like(x), x, poff, "sum")[0, 0] == 1.0
    assert R.sums_thr(np.abs(x) * np.sign(x), poff, ">", np.full((4, 1), -np.inf), 0.0)[0][0, 0] == 1.0


def test_float32_rounding_ties():
    """The float64 sum is rounded once, to nearest even: 1 + 2^-24 is a tie (-> 1), 1 + 2^-23 is exact, and a
    float32 running sum would lose both halves."""
    tie = np.float32(2.0 ** -24)
    x = np.array([[1.0, 1.0], [tie, tie], [0.0, tie]], np.float32)
    got = R.period_stat(x, np.array([0, 3]), "sum")[0]
    np.testing.assert_array_equal(got, np.array([1.0, 1.0 + 2.0 ** -23], np.float32))
    f32 = np.float32(0)
    for v in x[:, 1]:
        f32 = np.float32(f32 + v)
    assert f32 == 1.0


@pytest.mark.parametrize("v", [300.1, 271.35, 101325.0, 0.0, 1e-3, 3e38, 288.15])
def test_constant_cells_have_zero_variance(v):
    """Up to a year of a constant: q/n and mean^2 round to the same float64.  The one-pass formula has a limit:
    three years of 300.1 leave a residue (the sum of squares rounds on the way)."""
    for T in (1, 28, 90, 360, 365, 366):
        x = np.full((T, 1), v, np.float32)
        poff = np.array([0, T])
        assert R.period_stat(x, poff, "var")[0, 0] == 0.0, T
        assert R.period_stat(x, poff, "std")[0, 0] == 0.0, T
    if v == 300.1:
        assert R.period_stat(np.full((1096, 1), v, np.float32), np.array([0, 1096]), "var")[0, 0] > 0


def test_variance_formula_is_rounded_step_by_step():
    """var is fl(fl(q/n) - fl(m*m)), not the fused fl(fl(q/n) - m*m): on a large offset with a tiny spread the two
    differ in float32, which is what the GPU tests rely on to see a contracted formula."""
    rng = np.random.default_rng(7)
    x = (300.0 + 0.02 * rng.standard_normal((365, 64))).astype(np.float32)
    n, s, q, _, _ = R._moments(x)
    rule = R.period_stat(x, np.array([0, 365]), "var")[0]
    fused = []
    for j in range(x.shape[1]):
        m = s[j] / 365.0
        qn = q[j] / 365.0
        fused.append(float(Fraction(qn) - Fraction(m) * Fraction(m)))
        assert rule[j] == np.float32(max(qn - m * m, 0.0))         # Python floats: every operation rounded
    fused = np.maximum(np.array(fused), 0.0).astype(np.float32)
    assert (fused != rule).any()
