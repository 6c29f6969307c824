"""CPU checks of the window-sum rule reference (oracle window_stat_rule, spell_mask_rule, rolling_rule,
period_stat_rule) that tests/test_gpu_rolling_paths.py holds the rolling and spell kernels to: agreement with the
reference restatement where float32 and float64 sums agree, and known answers on hostile series."""
import numpy as np
import pytest

from oracle import xclim_oracle as O

POFF = np.array([0, 31, 59, 60, 181, 365, 425], np.int32)
REDUCERS = ["max", "min", "sum", "count", "mean", "std"]
FILL = np.float32(9.96921e36)


def _grid_field(seed, T=425, C=16):
    """0.5-grid precipitation: every float32 and float64 window sum is exact, so the rule and xarray agree."""
    rng = np.random.default_rng(seed)
    x = rng.gamma(0.4, 6.0, size=(T, C)).astype(np.float32)
    x[rng.random(x.shape) < 0.4] = 0.0
    x = (np.round(x * 2) / 2).astype(np.float32)
    x[rng.random(x.shape) < 0.03] = np.nan
    x[:, 0] = np.nan
    x[:, 1] = 1.0
    return x


@pytest.mark.parametrize("wstat", ["sum", "mean", "min", "max"])
@pytest.mark.parametrize("window", [1, 3, 7, 12])
def test_spell_rule_matches_reference(wstat, window):
    x = _grid_field(window)
    thr = 1.0 * window if wstat == "sum" else 1.0
    for op in (">", "<", ">=", "<=", "=="):     # "!=" differs near the series end: the reference pads with NaN
        mask = O.spell_mask_rule(x, window, wstat, op, thr).astype(np.float32)
        for before in (True, False):
            for red in REDUCERS:
                got = O.resample_and_rl(mask, before, O.rle_statistics, poff=POFF, reducer=red, window=1)
                exp = O.spell_length_statistics(x, thr, window, wstat, op, red, POFF, resample_before_rl=before)
                np.testing.assert_array_equal(np.asarray(got, np.float32), exp, err_msg=f"{op} {red} {before}")


@pytest.mark.parametrize("wstat", ["sum", "mean", "min", "max"])
@pytest.mark.parametrize("window,center", [(1, False), (3, True), (4, False), (9, True), (31, False)])
def test_rolling_rule_matches_reference(wstat, window, center):
    x = _grid_field(40 + window)
    vals = O.rolling_rule(x, window, wstat, center)
    np.testing.assert_array_equal(vals, O.rolling(x, window, wstat, center=center).astype(np.float32))
    for stat in ("sum", "mean", "min", "max", "std", "var", "count"):
        got = O.period_stat_rule(vals, POFF, stat)
        exp = O.select_rolling_resample_op(x.astype(np.float64), stat, window, POFF, window_center=center,
                                           window_op=wstat)
        # window means are not on the grid: the rule rounds each to float32 before the period sum
        if stat == "count" or (stat in ("sum", "min", "max") and wstat != "mean"):
            np.testing.assert_array_equal(got, exp.astype(np.float32), err_msg=stat)
        else:
            np.testing.assert_allclose(got, exp, rtol=1e-5, atol=1e-4, equal_nan=True, err_msg=stat)


def _series(bad):
    """40 days of 2.5 mm with ``bad`` {day: value}"""
    x = np.full((40, 1), 2.5, np.float32)
    for d, v in bad.items():
        x[d, 0] = v
    return x


def _sums(x, w=9):
    return O.window_stat_rule(x, w, "sum")[:, 0]


def test_known_answer_infinities():
    w, e = 9, np.arange(40)
    base = np.where(e >= w - 1, np.float32(22.5), np.nan)
    held = lambda d: (e >= d) & (e < d + w)                      # windows holding day d   # noqa: E731
    np.testing.assert_array_equal(_sums(_series({20: np.inf})), np.where(held(20), np.inf, base))
    np.testing.assert_array_equal(_sums(_series({20: -np.inf})), np.where(held(20), -np.inf, base))
    both = np.where(held(20) & held(23), np.nan, np.where(held(20), np.inf, np.where(held(23), -np.inf, base)))
    np.testing.assert_array_equal(_sums(_series({20: np.inf, 23: -np.inf})), both)
    # the mean and the extremes of a window holding an infinity
    x = _series({20: np.inf})
    np.testing.assert_array_equal(O.window_stat_rule(x, w, "mean")[:, 0][[19, 20, 28, 29]], [2.5, np.inf, np.inf, 2.5])
    np.testing.assert_array_equal(O.window_stat_rule(x, w, "max")[:, 0][[19, 28, 29]], [2.5, np.inf, 2.5])


def test_known_answer_fill_value():
    e = np.arange(40)
    got = _sums(_series({20: FILL}))
    held = (e >= 20) & (e < 29)
    np.testing.assert_array_equal(got, np.where(held, FILL, np.where(e >= 8, np.float32(22.5), np.nan)))
    # dry spells (9-day sum < 23 mm): every day but the filled one; two spells in the period, the longest 20 days
    mask = O.spell_mask_rule(_series({20: FILL}), 9, "sum", "<", 23.0)[:, 0]
    np.testing.assert_array_equal(mask, e != 20)
    poff = np.array([0, 40], np.int32)
    for red, v in (("count", 2), ("max", 20), ("min", 19), ("sum", 39)):
        got = O.resample_and_rl(mask[:, None].astype(np.float32), True, O.rle_statistics, poff=poff, reducer=red,
                                window=1)
        assert got[0, 0] == v, red


def test_known_answer_signed_zero_and_nan_run():
    z = np.full((20, 1), -0.0, np.float32)
    s = O.window_stat_rule(z, 5, "sum")[4:, 0]
    assert (s == 0).all() and not np.signbit(s).any()                    # the sum starts from +0.0
    assert np.signbit(O.window_stat_rule(z, 5, "min")[4:, 0]).all()
    x = _series({20: np.nan, 21: np.nan, 22: np.nan})
    e = np.arange(40)
    exp = np.where((e >= 20) & (e < 31) | (e < 8), np.nan, np.float32(22.5))
    np.testing.assert_array_equal(_sums(x), exp)
    # a NaN window only satisfies !=; every block holding day 20..22 fails "<"
    m = O.spell_mask_rule(x, 9, "sum", "<", 23.0)[:, 0]
    np.testing.assert_array_equal(m, ~((e >= 20) & (e <= 22)))
    assert O.spell_mask_rule(x, 9, "sum", "!=", 22.5)[:, 0][[12, 20, 30]].tolist() == [True, True, True]


def test_sum_is_sequential_float64():
    """Oldest first, one add at a time, rounded once: 1e8 + 1 + ... is not the pairwise sum of float32 values."""
    x = np.array([[1e8], [1.0], [1.0], [1.0], [-1e8]], np.float32)
    assert O.window_stat_rule(x, 5, "sum")[4, 0] == np.float32(3.0)
    x = np.array([[2.0 ** 60], [1.0], [-(2.0 ** 60)]], np.float32)
    assert O.window_stat_rule(x, 3, "sum")[2, 0] == 0.0                 # 2^60 + 1 rounds in float64
    assert O.period_stat_rule(np.array([[2.0 ** 60], [1.0], [-(2.0 ** 60)]], np.float32),
                              np.array([0, 3]), "sum")[0, 0] == 0.0
