"""GPU checks of every per-period float statistic against the float64 time-order rule (oracle/stat_rule.py), bit for
bit: float32 bits equal, any NaN equal to any NaN, -0 equal to +0.

The rule is what the kernels' comments promise: float64 sums and sums of squares added one value at a time in time
order, each result rounded to float32 once, var = q/n - mean^2 with every operation rounded, clamped at 0.  The
tolerances of the other GPU tests (1e-5 relative, 1e-4 absolute for std / var) pass a float32 sum, a pairwise sum
or a fused multiply-add in the variance; these tests do not.

Every cell carries one hostile pattern (``_hostile``): a large offset with a tiny spread, constant cells (whose
variance must be exactly 0), quantised values with ties at the thresholds, scattered NaN, an all-NaN period and a
period with one valid value, infinities (and +inf with -inf in one period: a NaN sum), +-3e38 (the float64 sum
overflows float32 on the final cast), subnormals and two columns whose float64 sum lands on a float32 rounding tie
or just past it.  Periods are raw offsets with one-step and empty periods and YS / MS / QS-DEC / YS-JUL on the
noleap, 360_day and standard calendars.  Layouts are 4 cells per lane (aligned, C % 4 == 0) and one cell per lane
(C % 4 != 0, or an offset column slice with ldx != C), C = 1, 127, 128, 129, and C >= 4096 for the bulk-copy
run-length kernel.
"""
import functools

import numpy as np
import pytest

from oracle import stat_rule as R
from oracle import xclim_oracle as O
from test_gpu_run_reducers import OPS, ROLL_CASES, SPELL_CASES

pytestmark = pytest.mark.gpu

STATS = R.STATS
RUN_REDUCERS = ("mean", "std")
TRANSFORMS = [("none", ">"), ("excess", ">"), ("excess", "<"), ("excess", ">="), ("excess", "<=")] + \
    [("where", op) for op in OPS]
THR = 1.0
TIE = np.float32(2.0 ** -24)          # 1 + 2^-24 is the float32 tie between 1 and 1 + 2^-23
N_PATTERNS = 16

# raw period offsets over 425 steps: one-step periods, and (EMPTY) periods with t0 == t1
RAW = np.array([0, 1, 2, 31, 59, 60, 61, 181, 365, 424, 425], np.int32)
EMPTY = np.array([0, 31, 31, 59, 60, 60, 181, 425, 425], np.int32)
CALENDARS = ("noleap", "360_day", "standard")
FREQS = ("YS", "MS", "QS-DEC", "YS-JUL")
PERIODS = ["raw"] + [f"{c}-{f}" for c in CALENDARS for f in FREQS]


@functools.lru_cache(maxsize=None)
def _axis(calendar):
    from xclim_b200 import TimeAxis
    # 3 years and 2 months from mid-November: partial periods at both ends, and Feb 29 2004 on the standard calendar
    return TimeAxis.daily("2003-11-15", {"noleap": 365, "360_day": 360, "standard": 365}[calendar] * 3 + 60, calendar)


def _periods(name):
    """(T, poff) of a period case"""
    if name == "raw":
        return 425, RAW
    if name == "empty":
        return 425, EMPTY
    cal, freq = name.split("-", 1)
    ta = _axis(cal)
    return len(ta), np.asarray(ta.period_offsets(freq), np.int32)


def _hostile(T, C, poff, seed):
    """(T, C) float32: column c carries pattern (c + seed) % N_PATTERNS."""
    rng = np.random.default_rng(seed)
    x = np.empty((T, C), np.float32)
    n = rng.standard_normal((T, C))
    q = np.round(rng.gamma(0.4, 6.0, (T, C)) * 2) / 2
    q[rng.random((T, C)) < 0.4] = 0.0
    starts = [int(s) for s, e in O._groups(poff) if e > s]
    for c in range(C):
        k = (c + seed) % N_PATTERNS
        if k == 0:
            v = 300.0 + 0.02 * n[:, c]                  # a tropical SST: large offset, tiny spread
        elif k == 1:
            v = 101325.0 + n[:, c]                      # surface pressure in Pa
        elif k == 2:
            v = np.full(T, 300.1)                       # constant cells: var exactly 0
        elif k == 3:
            v = np.full(T, 271.35)
        elif k == 4:
            v = q[:, c]                                 # quantised, ties with THR
        elif k == 5:
            v = np.where(rng.random(T) < 0.3, np.nan, q[:, c])      # scattered NaN
        elif k == 6:
            v = 280.0 + 3.0 * n[:, c]                   # an all-NaN first period, one valid value in the second
            v[poff[0]:poff[1]] = np.nan
            if len(poff) > 2 and poff[2] > poff[1]:
                v[poff[1]:poff[2]] = np.nan
                v[(poff[1] + poff[2]) // 2] = 281.5
        elif k == 7:
            v = np.where(rng.random(T) < 0.02, np.inf, 280.0 + 3.0 * n[:, c])
        elif k == 8:
            v = np.where(rng.random(T) < 0.02, -np.inf, q[:, c])
        elif k == 9:                                    # +inf and -inf in the same periods: NaN sums and means
            v = q[:, c].copy()
            for s in starts:
                v[s] = np.inf
                v[min(s + 1, T - 1)] = -np.inf
        elif k == 10:
            v = np.where(rng.random(T) < 0.8, 3e38, -3e38)          # the float64 sum overflows float32
        elif k == 11:
            v = np.where(rng.random(T) < 0.5, 3e38, 1.0)
        elif k == 12:                                   # subnormals
            v = (rng.integers(-2 ** 20, 2 ** 20, T) * 2.0 ** -149) * (rng.random(T) < 0.7)
        elif k in (13, 14):                             # the float64 sum lands on a float32 tie (13) or just past it
            v = np.zeros(T)
            for s in starts:
                v[s] = 1.0
                v[min(s + 1, T - 1)] = TIE
                if k == 14:
                    v[min(s + 2, T - 1)] = TIE
        else:
            v = 288.15 + 0.5 * np.round(4 * n[:, c]) / 4
        x[:, c] = np.asarray(v, np.float64).astype(np.float32)
    return x


# ----------------------------------------------------------------------------------------------- comparison
def _same(got, exp, msg):
    got = np.asarray(got.cpu().numpy() if hasattr(got, "cpu") else got, np.float32)
    exp = np.asarray(exp, np.float32)
    assert got.shape == exp.shape, f"{msg}: shape {got.shape} != {exp.shape}"
    ok = (got == exp) | (np.isnan(got) & np.isnan(exp))
    if not ok.all():
        bad = np.argwhere(~ok)[:6]
        detail = ", ".join(f"{tuple(int(i) for i in b)}: {got[tuple(b)]!r} != {exp[tuple(b)]!r}" for b in bad)
        raise AssertionError(f"{msg}: {int((~ok).sum())} of {ok.size} differ from the rule ({detail})")


def _views(x, layout):
    """(T, C) device view of x: 'aligned' (4 cells per lane when C % 4 == 0) or 'slice' (an offset column slice of a
    wider buffer, ldx = C + 3: one cell per lane)."""
    import torch
    a = torch.from_numpy(x).cuda()
    if layout == "aligned":
        return a
    buf = torch.full((x.shape[0], x.shape[1] + 3), float("nan"), device="cuda")
    buf[:, 1:x.shape[1] + 1] = a
    return buf[:, 1:x.shape[1] + 1]


def _valid(x, poff):
    return np.stack([(~np.isnan(x[s:e])).sum(0) for s, e in O._groups(poff)]).astype(np.int32)


# ----------------------------------------------------------------------------------------------- period_reduce
def _check_period_reduce(x, poff, layout, tag):
    from xclim_b200 import _lib, device
    xv = _views(x, layout)
    valid_exp = _valid(x, poff)
    for i, (kind, op) in enumerate(TRANSFORMS):
        tf = {"none": _lib.TF_NONE, "excess": _lib.TF_EXCESS, "where": _lib.TF_WHERE}[kind]
        for j, stat in enumerate(STATS):
            want_valid = (i + j) % 2 == 0
            exp = R.period_stat(x, poff, stat, kind, op, THR)
            got, valid = device.period_reduce(xv, poff, _lib.STATS[stat], tf, _lib.OPS[op], THR, want_valid)
            _same(got, exp, f"{tag} {layout} {stat} {kind} {op}")
            if want_valid:
                np.testing.assert_array_equal(valid.cpu().numpy(), valid_exp, err_msg=f"{tag} valid")


@pytest.mark.parametrize("layout", ["aligned", "slice"])
@pytest.mark.parametrize("periods", PERIODS + ["empty"])
def test_period_reduce(cuda, periods, layout):
    T, poff = _periods(periods)
    _check_period_reduce(_hostile(T, 64, poff, 0), poff, layout, periods)


@pytest.mark.parametrize("C", [1, 127, 128, 129])
@pytest.mark.parametrize("periods", ["raw", "standard-QS-DEC"])
def test_period_reduce_widths(cuda, periods, C):
    T, poff = _periods(periods)
    _check_period_reduce(_hostile(T, C, poff, C), poff, "aligned", f"{periods} C={C}")


# ----------------------------------------------------------------------------------------------- rolling
@pytest.mark.parametrize("wstat,window,center", ROLL_CASES)
@pytest.mark.parametrize("periods", ["raw", "empty", "standard-MS", "360_day-YS-JUL"])
def test_rolling_period_reduce(cuda, periods, wstat, window, center):
    from xclim_b200 import _lib, device
    T, poff = _periods(periods)
    x = _hostile(T, 64, poff, window)
    vals = O.rolling_rule(x, window, wstat, center)
    views = [(name, _views(x, name)) for name in ("aligned", "slice")]
    for stat in STATS:
        exp = R.period_stat(vals, poff, stat)
        for name, xv in views:
            got = device.rolling_period_reduce(xv, poff, window, _lib.STATS[wstat], center, _lib.STATS[stat])
            _same(got, exp, f"{periods} {wstat}{window} center={center} {stat} {name}")


@pytest.mark.parametrize("wstat,window,center", ROLL_CASES)
def test_rolling_period_reduce_sel(cuda, wstat, window, center):
    from xclim_b200 import _lib, device
    T, poff = _periods("noleap-QS-DEC")
    x = _hostile(T, 48, poff, 3)
    keep = np.asarray(_axis("noleap").month) % 3 != 1
    keep[poff[2]:poff[3]] = False                   # a period that keeps nothing
    vals = np.where(keep[:, None], O.rolling_rule(x, window, wstat, center), np.float32(np.nan))
    for stat in STATS:
        exp = R.period_stat(vals, poff, stat)
        for name in ("aligned", "slice"):
            got = device.rolling_period_reduce_sel(_views(x, name), poff, window, _lib.STATS[wstat], center,
                                                   _lib.STATS[stat], keep.astype(np.uint8))
            _same(got, exp, f"{wstat}{window} center={center} {stat} {name}")


# ----------------------------------------------------------------------------------------------- daily range
def _range_pair(T, C, poff, seed):
    rng = np.random.default_rng(seed + 100)
    hi = _hostile(T, C, poff, seed)
    lo = (hi - np.float32(5.0) - np.abs(3.0 * rng.standard_normal((T, C))).astype(np.float32)).astype(np.float32)
    lo[rng.random((T, C)) < 0.02] = np.nan
    lo[:, ::5] = _hostile(T, C, poff, seed + 7)[:, ::5]          # cancellation and infinities on both sides
    return lo, hi


def _pair_views(a, b, layout):
    """(T, C) device views of two inputs with one row stride: contiguous, or offset column slices (ldx = C + 3)."""
    import torch
    if layout == "aligned":
        return _views(a, "aligned"), _views(b, "aligned")
    T, C = a.shape
    buf = torch.full((2, T, C + 3), float("nan"), device="cuda")
    buf[0, :, 1:C + 1] = torch.from_numpy(a).cuda()
    buf[1, :, 1:C + 1] = torch.from_numpy(b).cuda()
    return buf[0, :, 1:C + 1], buf[1, :, 1:C + 1]


@pytest.mark.parametrize("C", [1, 129, 128])
@pytest.mark.parametrize("periods", ["raw", "empty", "noleap-MS", "standard-YS", "360_day-QS-DEC"])
def test_period_range_stat(cuda, periods, C):
    from xclim_b200 import _lib, device
    T, poff = _periods(periods)
    lo, hi = _range_pair(T, C, poff, C)
    for name in ("aligned", "slice"):
        lv, hv = _pair_views(lo, hi, name)
        for stat in STATS:
            _same(device.period_range_stat(lv, hv, poff, _lib.STATS[stat]), R.range_stat(lo, hi, poff, stat),
                  f"{periods} {stat} {name}")
        _same(device.period_range_stat(lv, hv, poff, _lib.STATS["mean"], variability=True),
              R.range_stat(lo, hi, poff, "mean", variability=True), f"{periods} variability {name}")


# ----------------------------------------------------------------------------------------------- run reducers
def _run_exp(mask, poff, red, window, before):
    return O.resample_and_rl(mask, before, R.run_stat, poff=poff, reducer=red, window=window)


@pytest.mark.parametrize("before", [True, False])
@pytest.mark.parametrize("periods", ["raw", "noleap-YS", "standard-MS", "360_day-YS-JUL"])
def test_period_runstat(cuda, periods, before):
    from xclim_b200 import _lib, device
    T, poff = _periods(periods)
    x = _hostile(T, 64, poff, 5)
    views = [(name, _views(x, name)) for name in ("aligned", "slice")]
    for i, op in enumerate(OPS):
        mask = O.compare(x, op, THR)
        for window in (1, 3):
            for red in RUN_REDUCERS:
                exp = _run_exp(mask, poff, red, window, before)
                for name, xv in views:
                    got, _ = device.period_runstat(xv, poff, _lib.OPS[op], THR, _lib.RL_REDUCERS[red], window, before,
                                                   want_valid=(i % 2 == 0))
                    _same(got, exp, f"{periods} {op} {red} w={window} before={before} {name}")


@pytest.mark.parametrize("per_lane", [False, True])
def test_period_runstat_wide(cuda, monkeypatch, per_lane):
    """C >= 4096, aligned, runs cut at the period edges: the mean reducer goes to the bulk-copy kernel (the std
    reducer and XCLIM_B200_RUNSTAT_V1 to the per-lane kernel); 4100 cells leave a partial second tile."""
    from xclim_b200 import _lib, device
    if per_lane:
        monkeypatch.setenv("XCLIM_B200_RUNSTAT_V1", "1")
    else:
        monkeypatch.delenv("XCLIM_B200_RUNSTAT_V1", raising=False)
    T, poff = _periods("standard-YS")
    x = _hostile(T, 4100, poff, 9)
    xv = _views(x, "aligned")
    for op in (">", "<=", "!="):
        mask = O.compare(x, op, THR)
        for window in (1, 4):
            for red in RUN_REDUCERS:
                exp = _run_exp(mask, poff, red, window, True)
                for want_valid in (False, True):
                    got, valid = device.period_runstat(xv, poff, _lib.OPS[op], THR, _lib.RL_REDUCERS[red], window,
                                                       True, want_valid=want_valid)
                    _same(got, exp, f"{op} {red} w={window}")
                    if want_valid:
                        np.testing.assert_array_equal(valid.cpu().numpy(), _valid(x, poff))


def _doy_table(rng, x, doy, n_doy):
    """float64 per-doy thresholds: data values (ties) and values between two float32s"""
    tab = np.full((n_doy, x.shape[1]), 280.0)
    for d in range(1, n_doy + 1):
        rows = np.nonzero(doy == d)[0]
        if rows.size:
            tab[d - 1] = np.nan_to_num(x[rows[0]].astype(np.float64), nan=280.0, posinf=280.0, neginf=280.0)
    return tab + np.where(rng.random(tab.shape) < 0.5, 0.0, rng.standard_normal(tab.shape) * 1e-6)


@pytest.mark.parametrize("before", [True, False])
@pytest.mark.parametrize("calendar", CALENDARS)
def test_doy_runstat(cuda, calendar, before):
    import torch
    from xclim_b200 import _lib, device
    ta = _axis(calendar)
    T, doy = len(ta), np.asarray(ta.doy)
    rng = np.random.default_rng(11)
    x = _hostile(T, 68, np.array([0, T]), 2)
    tab = _doy_table(rng, x, doy, int(ta.max_doy))
    tab_d = torch.from_numpy(tab).cuda()
    for freq in ("YS", "MS"):
        poff = ta.period_offsets(freq)
        for op in (">", "<", ">=", "<="):
            mask = O.compare(x, op, tab[doy - 1])
            for window in (1, 3):
                for red in RUN_REDUCERS:
                    exp = _run_exp(mask, poff, red, window, before)
                    for name in ("aligned", "slice"):
                        got, _ = device.doy_runstat(_views(x, name), poff, doy, tab_d, _lib.OPS[op],
                                                    _lib.RL_REDUCERS[red], window, before, want_valid=True)
                        _same(got, exp, f"{freq} {op} {red} w={window} {name}")


@pytest.mark.parametrize("var_any", [False, True])
@pytest.mark.parametrize("before", [True, False])
def test_period_runstat2(cuda, before, var_any):
    from xclim_b200 import _lib, device
    T, poff = _periods("noleap-MS")
    x1, x2 = _hostile(T, 64, poff, 1), _hostile(T, 64, poff, 6)
    for layout in ("aligned", "slice"):
        a, b = _pair_views(x1, x2, layout)
        for op1, op2 in ((">", ">"), ("<=", "!="), ("==", ">=")):
            c1, c2 = O.compare(x1, op1, THR), O.compare(x2, op2, 2.0)
            mask = (c1 | c2) if var_any else (c1 & c2)
            for window in (1, 3):
                for red in RUN_REDUCERS:
                    got = device.period_runstat2(a, b, poff, _lib.OPS[op1], THR, _lib.OPS[op2], 2.0,
                                                 _lib.RL_REDUCERS[red], window, before, var_any)
                    _same(got, _run_exp(mask, poff, red, window, before), f"{layout} {op1}{op2} {red} w={window}")


@pytest.mark.parametrize("min_gap", [2, 3])
def test_period_runstat_gap(cuda, min_gap):
    from xclim_b200 import _lib, device
    T, poff = _periods("standard-QS-DEC")
    x = _hostile(T, 64, poff, 4)
    xv = _views(x, "aligned")
    for op in OPS:
        m = O.compare(x, op, THR)
        filled = O.runs_with_holes(m, 1, ~m, min_gap).astype(np.float32)
        for window in (1, 3):
            for red in RUN_REDUCERS:
                got = device.period_runstat_gap(xv, poff, _lib.OPS[op], THR, _lib.RL_REDUCERS[red], min_gap, window)
                _same(got, _run_exp(filled, poff, red, window, True), f"{op} {red} w={window}")


@pytest.mark.parametrize("wstat,window", SPELL_CASES)
@pytest.mark.parametrize("before", [True, False])
def test_spell_runstat(cuda, wstat, window, before):
    from xclim_b200 import _lib, device
    T, poff = _periods("noleap-MS")
    x = _hostile(T, 64, poff, window)
    thr = THR * window if wstat == "sum" else THR
    views = [(name, _views(x, name)) for name in ("aligned", "slice")]
    for op in OPS:
        mask = O.spell_mask_rule(x, window, wstat, op, thr).astype(np.float32)
        for red in RUN_REDUCERS:
            exp = _run_exp(mask, poff, red, 1, before)
            for name, xv in views:
                got = device.spell_runstat(xv, poff, window, _lib.STATS[wstat], _lib.OPS[op], thr,
                                           _lib.RL_REDUCERS[red], before)
                _same(got, exp, f"{wstat}{window} {op} {red} before={before} {name}")


# ----------------------------------------------------------------------------------------------- run sums
@pytest.mark.parametrize("before", [True, False])
@pytest.mark.parametrize("periods", ["raw", "noleap-YS", "360_day-MS", "standard-YS-JUL"])
def test_period_run_maxsum(cuda, periods, before):
    from xclim_b200 import _lib, device
    T, poff = _periods(periods)
    x = _hostile(T, 64, poff, 8)
    views = [(name, _views(x, name)) for name in ("aligned", "slice")]
    for op in (">", "<", ">=", "<="):
        for thr in (THR, 300.0):
            for window in (1, 3):
                exp = R.run_maxsum(x, poff, op, thr, window, before)
                for name, xv in views:
                    got = device.period_run_maxsum(xv, poff, _lib.OPS[op], thr, window, before)
                    _same(got, exp, f"{periods} {op} thr={thr} w={window} before={before} {name}")


@pytest.mark.parametrize("table", ["doy", "cell"])
@pytest.mark.parametrize("calendar", CALENDARS)
def test_period_sums_thr(cuda, calendar, table):
    import torch
    from xclim_b200 import _lib, device
    ta = _axis(calendar)
    T, doy = len(ta), np.asarray(ta.doy)
    rng = np.random.default_rng(13)
    x = _hostile(T, 132, np.array([0, T]), 3)
    if table == "doy":
        tab = _doy_table(rng, np.where(np.abs(x) < 1e30, x, np.float32(1.0)), doy, int(ta.max_doy))
        tab[:, ::7] = 1.0                               # exactly at the quantised values
        rows = tab[doy - 1]
    else:
        tab = np.where(rng.random((1, x.shape[1])) < 0.5, 1.0, 0.5 + 1e-9)
        rows = tab
    tab_d = torch.from_numpy(tab).cuda()
    for freq in FREQS:
        poff = ta.period_offsets(freq)
        for op in (">", ">="):
            exp_thr, exp_wet = R.sums_thr(x, poff, op, rows, 1.0)
            for name in ("aligned", "slice"):
                s_thr, s_wet = device.period_sums_thr(_views(x, name), poff, _lib.OPS[op], tab_d, 1.0,
                                                      doy_index=doy if table == "doy" else None)
                _same(s_thr, exp_thr, f"{freq} {op} thr {name}")
                _same(s_wet, exp_wet, f"{freq} {op} wet {name}")


# ----------------------------------------------------------------------------------------------- cross paths
@pytest.mark.parametrize("layout", ["aligned", "slice"])
@pytest.mark.parametrize("periods", ["raw", "standard-MS"])
def test_statistic_copies_agree(cuda, periods, layout):
    """One series through every copy of the statistic formula: period_reduce_kernel's, StatAcc's in the rolling
    kernels (window 1, window statistic max: the value itself) and in the daily-range kernel (lo = 0), and the rule:
    bit-identical."""
    from xclim_b200 import _lib, device
    T, poff = _periods(periods)
    x = _hostile(T, 128, poff, 0)
    zeros, xv = _pair_views(np.zeros_like(x), x, layout)
    for stat in STATS:
        code = _lib.STATS[stat]
        exp = R.period_stat(x, poff, stat)
        outs = {"period_reduce": device.period_reduce(xv, poff, code)[0],
                "rolling w=1": device.rolling_period_reduce(xv, poff, 1, _lib.STATS["max"], False, code),
                "range lo=0": device.period_range_stat(zeros, xv, poff, code)}
        for name, got in outs.items():
            _same(got, exp, f"{stat} {name} {layout}")
