"""GPU parity of the run-length reducers and the per-period statistics on every kernel path the dispatch picks.

Every run-length entry point runs all six reducers, every rolling / reduce entry point all seven statistics, on
data with NaN, a cell with no runs, a cell sitting on the threshold and runs across period edges, under all six
operators.  Integer-valued results match the oracle exactly, mean and std at 1e-5 relative.  The run-length
reduction is the same integer arithmetic on every path, so the paths that can see the same input must also agree
with each other bit for bit.

The dispatch is decided by the cell layout (``C % 4``, row stride and alignment: an offset column slice takes the
one-cell-per-lane paths), the window, the window statistic and the shared-memory ring size (w * 2 kB <= 160 kB).
"""
import numpy as np
import pytest

import fake_device as F
from oracle import xclim_oracle as O

pytestmark = pytest.mark.gpu

OPS = [">", "<", ">=", "<=", "==", "!="]
REDUCERS = ["max", "min", "sum", "count", "mean", "std"]
STATS = ["sum", "mean", "min", "max", "std", "var", "count"]
POFF = np.array([0, 31, 59, 60, 181, 365, 425], np.int32)   # includes a one-step period
T, C = 425, 24
THR = 1.0


def _field(seed):
    rng = np.random.default_rng(seed)
    x = rng.gamma(0.4, 6.0, size=(T, C)).astype(np.float32)
    x[rng.random(x.shape) < 0.4] = 0.0
    x = np.round(x * 2) / 2                       # many exact ties with the thresholds
    x[rng.random(x.shape) < 0.03] = np.nan
    x[:, 0] = np.nan                              # no runs at all (but one long != run)
    x[:, 1] = THR                                 # on the threshold everywhere
    x[20:80, 2] = 5.0                             # runs across the period edges at 31, 59 and 60
    x[25:70, 3] = 0.0
    x[40, 3] = np.nan                             # ... one of them cut by a NaN
    x[:3, 4] = 5.0; x[-3:, 4] = 5.0               # runs open at the series start and end
    return x.astype(np.float32)


def _views(x):
    """The same cells as an aligned tensor (4 cells per thread) and as an offset column slice (ldx = C + 1,
    4-byte offset: one cell per lane)."""
    import torch
    a = torch.from_numpy(x).cuda()
    buf = torch.zeros((x.shape[0], x.shape[1] + 1), dtype=torch.float32, device=a.device)
    buf[:, 1:] = a
    return a, buf[:, 1:]


def _check_runs(got, exp, red, msg):
    if red in ("mean", "std"):
        np.testing.assert_allclose(got, exp, rtol=1e-5, atol=0, err_msg=msg)
    else:
        np.testing.assert_array_equal(got, exp, err_msg=msg)


def _check_stat(got, exp, stat, msg):
    if stat == "count":
        np.testing.assert_array_equal(got, exp, err_msg=msg)
    else:   # float reductions: 1e-5 relative; std / var one-pass in float64 (1e-4 absolute, as elsewhere)
        np.testing.assert_allclose(got, exp, rtol=1e-5, atol=1e-4 if stat in ("std", "var") else 0, equal_nan=True,
                                   err_msg=msg)


def _same_bits(outs, msg):
    for o in outs[1:]:
        np.testing.assert_array_equal(o.view(np.uint32), outs[0].view(np.uint32), err_msg=msg)


# ---------------------------------------------------------------------------------------- period_runstat_kernel
@pytest.mark.parametrize("window", [1, 3])   # max at window 1 takes the FASTMAX running form
@pytest.mark.parametrize("before", [True, False])
def test_period_runstat_vec4_vec1(cuda, window, before):
    from xclim_b200 import _lib, device
    x = _field(1)
    views = _views(x)
    for op in OPS:
        for red in REDUCERS:
            args = (POFF, _lib.OPS[op], THR, _lib.RL_REDUCERS[red], window, before)
            exp = F.period_runstat(x, *args)[0].numpy()
            got = [device.period_runstat(v, *args, want_valid=before)[0].cpu().numpy() for v in views]
            msg = f"{op} {red} w={window} before={before}"
            _check_runs(got[0], exp, red, msg)
            _same_bits(got, msg)


# ----------------------------------------------------------------------------------------- period_run_maxsum_kernel
@pytest.mark.parametrize("window", [1, 3])
@pytest.mark.parametrize("before", [True, False])
def test_period_run_maxsum_vec4_vec1(cuda, window, before):
    from xclim_b200 import _lib, device
    x = _field(11)
    views = _views(x)
    for op in (">", "<"):
        args = (POFF, _lib.OPS[op], THR, window, before)
        exp = F.period_run_maxsum(x, *args).numpy()
        got = [device.period_run_maxsum(v, *args).cpu().numpy() for v in views]
        msg = f"{op} w={window} before={before}"
        np.testing.assert_allclose(got[0], exp, rtol=1e-5, atol=1e-6, err_msg=msg)
        _same_bits(got, msg)


# --------------------------------------------------------------------- spell_sumw / spell_runstat4 / spell_runstat
# (window statistic, window): aligned kernel / offset-slice kernel
SPELL_CASES = [
    pytest.param("sum", 2, id="sumw-sum2/runstat"),
    pytest.param("sum", 5, id="sumw-sum5/runstat"),
    pytest.param("mean", 3, id="sumw-mean3/runstat"),
    pytest.param("mean", 8, id="sumw-mean8/runstat"),
    pytest.param("min", 3, id="runstat4-min3/runstat"),
    pytest.param("max", 4, id="runstat4-max4/runstat"),
    pytest.param("sum", 9, id="runstat4-sum9/runstat"),
    pytest.param("mean", 12, id="runstat4-mean12/runstat"),
    pytest.param("sum", 90, id="runstat-sum90/runstat"),   # the ring does not fit shared memory
]


@pytest.mark.parametrize("wstat,window", SPELL_CASES)
@pytest.mark.parametrize("before", [True, False])
def test_spell_runstat_paths(cuda, wstat, window, before):
    from xclim_b200 import _lib, device
    x = _field(2)
    views = _views(x)
    thr = THR * window if wstat == "sum" else THR
    for op in OPS:
        for red in REDUCERS:
            args = (POFF, window, _lib.STATS[wstat], _lib.OPS[op], thr, _lib.RL_REDUCERS[red], before)
            exp = F.spell_runstat(x, *args).numpy()
            got = [device.spell_runstat(v, *args).cpu().numpy() for v in views]
            msg = f"{wstat}{window} {op} {red} before={before}"
            if op != "!=":   # the reference counts windows that run off the series as NaN, and NaN != thr
                _check_runs(got[0], exp, red, msg)
            _same_bits(got, msg)


# ------------------------------------------------------------------------------------------ period_runstat2_kernel
@pytest.mark.parametrize("op1,op2", [pytest.param(">", ">", id="GTGT"), ("<=", "!="), ("==", ">="), ("<", "=="),
                                     ("!=", "<")])
@pytest.mark.parametrize("var_any", [False, True])
@pytest.mark.parametrize("before", [True, False])
def test_period_runstat2_vec4_vec1(cuda, op1, op2, var_any, before):
    from xclim_b200 import _lib, device
    x1, x2 = _field(3), _field(4)
    v1, v2 = _views(x1), _views(x2)
    for window in (1, 3):
        for red in REDUCERS:
            args = (POFF, _lib.OPS[op1], THR, _lib.OPS[op2], 2.0, _lib.RL_REDUCERS[red], window, before, var_any)
            exp = F.period_runstat2(x1, x2, *args).numpy()
            got = [device.period_runstat2(a, b, *args).cpu().numpy() for a, b in zip(v1, v2)]
            msg = f"{red} w={window}"
            _check_runs(got[0], exp, red, msg)
            _same_bits(got, msg)


# -------------------------------------------------------------------------------------- period_runstat_gap_kernel
@pytest.mark.parametrize("min_gap", [2, 3, 5])
def test_period_runstat_gap(cuda, min_gap):
    import torch
    from xclim_b200 import _lib, device
    x = _field(5)
    xd = torch.from_numpy(x).cuda()
    for op in OPS:
        for window in (1, 3):
            for red in REDUCERS:
                args = (POFF, _lib.OPS[op], THR, _lib.RL_REDUCERS[red], min_gap, window)
                exp = F.period_runstat_gap(x, *args).numpy()
                got = device.period_runstat_gap(xd, *args).cpu().numpy()
                _check_runs(got, exp, red, f"{op} {red} w={window}")


def test_run_length_paths_agree(cuda):
    """One window-1 mask through every run-length kernel: bit-identical results for all six reducers."""
    from xclim_b200 import _lib, device
    x = _field(6)
    views = _views(x)
    ones = _views(np.ones_like(x))
    gt = _lib.OPS[">"]
    for op in OPS:
        for before in (True, False):
            for window in (1, 3):
                for red in REDUCERS:
                    o, r = _lib.OPS[op], _lib.RL_REDUCERS[red]
                    outs = [device.period_runstat(v, POFF, o, THR, r, window, before)[0] for v in views]
                    outs += [device.period_runstat2(v, w1, POFF, o, THR, _lib.OPS["=="], 1.0, r, window, before)
                             for v, w1 in zip(views, ones)]
                    if op == ">":
                        outs += [device.period_runstat2(v, w1, POFF, gt, THR, gt, 0.0, r, window, before)
                                 for v, w1 in zip(views, ones)]
                    if window == 1:   # a window-1 "max" window statistic is the value itself
                        outs += [device.spell_runstat(v, POFF, 1, _lib.STATS["max"], o, THR, r, before) for v in views]
                    if before:
                        outs.append(device.period_runstat_gap(views[0], POFF, o, THR, r, 1, window))
                    _same_bits([t.cpu().numpy() for t in outs], f"{op} {red} w={window} before={before}")


# ------------------------------------------------------------------ rolling_sumw / rolling_period_reduce(4) / _sel
# (window statistic, window, center): kernel of the aligned layout / kernel of the offset slice
ROLL_CASES = [
    pytest.param("sum", 3, False, id="sumw-sum3/reduce-slide"),
    pytest.param("mean", 5, True, id="sumw-mean5/reduce-slide"),
    pytest.param("sum", 1, False, id="reduce4-sum1/reduce-slide"),
    pytest.param("sum", 9, True, id="reduce4-sum9/reduce-slide"),
    pytest.param("max", 4, False, id="reduce4-max4/reduce-rescan"),
    pytest.param("min", 7, True, id="reduce4-min7/reduce-rescan"),
    pytest.param("mean", 91, True, id="reduce-mean91/reduce-slide"),   # the ring does not fit shared memory
]


@pytest.mark.parametrize("wstat,window,center", ROLL_CASES)
def test_rolling_period_reduce_paths(cuda, wstat, window, center):
    from xclim_b200 import _lib, device
    x = _field(7)
    views = _views(x)
    for stat in STATS:
        args = (POFF, window, _lib.STATS[wstat], center, _lib.STATS[stat])
        exp = F.rolling_period_reduce(x, *args).numpy()
        for v, name in zip(views, ("aligned", "slice")):
            _check_stat(device.rolling_period_reduce(v, *args).cpu().numpy(), exp, stat, f"{stat} {name}")


@pytest.mark.parametrize("wstat,window,center", [("sum", 3, False), ("mean", 5, True), ("min", 1, False),
                                                 ("max", 7, True)])
def test_rolling_period_reduce_sel(cuda, wstat, window, center):
    from xclim_b200 import _lib, device
    x = _field(8)
    rng = np.random.default_rng(9)
    keep = ((np.arange(T) % 365 >= 90) & (np.arange(T) % 365 < 250)) | (rng.random(T) < 0.1)
    keep[59] = False                              # the one-step period keeps nothing
    for stat in STATS:
        args = (POFF, window, _lib.STATS[wstat], center, _lib.STATS[stat], keep.astype(np.uint8))
        exp = F.rolling_period_reduce_sel(x, *args).numpy()
        for v in _views(x):
            _check_stat(device.rolling_period_reduce_sel(v, *args).cpu().numpy(), exp, stat, stat)


# -------------------------------------------------------------------------------------------- period_reduce_kernel
@pytest.mark.parametrize("transform,op", [("none", ">"), ("excess", ">"), ("excess", "<")] +
                         [("where", op) for op in OPS])
def test_period_reduce_paths(cuda, transform, op):
    from xclim_b200 import _lib, device
    x = _field(10)
    tf = {"none": _lib.TF_NONE, "excess": _lib.TF_EXCESS, "where": _lib.TF_WHERE}[transform]
    if transform == "excess":   # (x - t).clip(0) / (t - x).clip(0) in float32, NaN kept
        d = (x - np.float32(THR)) if op == ">" else (np.float32(THR) - x)
        y = np.where(np.isnan(d), np.nan, np.maximum(d, 0)).astype(np.float64)
    valid_exp = np.stack([(~np.isnan(x[s:e])).sum(0) for s, e in O._groups(POFF)])
    for stat in STATS:
        if transform == "excess":
            exp = O.resample_reduce(y, POFF, stat)
        else:
            exp = F.period_reduce(x, POFF, _lib.STATS[stat], tf, _lib.OPS[op], THR)[0].numpy()
        for v, name in zip(_views(x), ("vec4", "vec1")):
            for want_valid in (False, True):
                got, valid = device.period_reduce(v, POFF, _lib.STATS[stat], tf, _lib.OPS[op], THR, want_valid)
                _check_stat(got.cpu().numpy(), exp, stat, f"{stat} {name} valid={want_valid}")
                if want_valid:
                    np.testing.assert_array_equal(valid.cpu().numpy(), valid_exp)
