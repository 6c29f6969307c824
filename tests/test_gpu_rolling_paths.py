"""GPU parity of every rolling-window and spell kernel behind xc_rolling_period_reduce_f32, xc_spell_runstat_f32
and xc_spell_mask_f32 against the window-sum rule (oracle window_stat_rule: the float64 sum of the window in
time order, NaN if any value is NaN, rounded once to float32).

Each case names the kernel instances it is meant to reach (the launch plans the launchers execute),
checks them against the launches torch.profiler records, and compares the outputs with the rule: spell run
statistics and rolling sum / min / max / count exactly, means, std and var at the tolerances of
test_gpu_run_reducers.py.  Paths that see the same cells must agree: spell outputs bit for bit, rolling outputs by
value (the sign of a zero window sum is not part of the rule: the register kernels start from the oldest value).

The data are continuous gamma precipitation with NaN, a NaN run, an all-NaN cell, a constant cell whose window
statistic is the threshold and thresholds equal to window statistics of the data (ties), and hostile cells early
in a period: +inf, -inf, +inf and -inf in one window, the netCDF default fill 9.96921e36 and a run of -0.0.  A
sliding float64 sum that is not checked for exactness turns every later window of the period into NaN after an
infinity, and loses the values that the fill value absorbed.
"""
import numpy as np
import pytest

from oracle import xclim_oracle as O
import dispatch_host_build as H

pytestmark = pytest.mark.gpu

OPS = [">", "<", ">=", "<=", "==", "!="]
REDUCERS = ["max", "min", "sum", "count", "mean", "std"]
STATS = ["sum", "mean", "min", "max", "std", "var", "count"]
WSTATS = ["sum", "mean", "min", "max"]
RL = {"max": 0, "min": 1, "sum": 2, "count": 3, "mean": 4, "std": 5}
ST = {"sum": 0, "mean": 1, "min": 2, "max": 3, "std": 4, "var": 5, "count": 6}
OPC = {">": 0, "<": 1, ">=": 2, "<=": 3, "==": 4, "!=": 5}
FILL = np.float32(9.96921e36)
WINDOWS = [1, 2, 3, 4, 5, 6, 7, 8, 9, 12, 31, 80, 81]

_NOLEAP = np.array([31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31])
P_SMALL = np.array([0, 31, 59, 60, 62, 181, 365, 425], np.int32)        # a one-step and a two-step period
P_MS = np.concatenate([[0], np.cumsum(np.tile(_NOLEAP, 2))]).astype(np.int32)           # 730 days
P_QS = np.array([0, 59, 151, 243, 334, 424, 516, 608, 699, 730], np.int32)             # QS-DEC on Jan 1st
P_YS = (np.arange(31) * 365).astype(np.int32)                                           # 10950 days


# ------------------------------------------------------------------------------------------------- data
def _hostile(x, cells, days):
    """+inf, -inf, +inf then -inf two steps later, the fill value, a run of -0.0 and a NaN run, in ``cells``
    (six columns) at each of ``days``."""
    for d in days:
        x[d, cells[0]] = np.inf
        x[d, cells[1]] = -np.inf
        x[d, cells[2]] = np.inf
        x[d + 2, cells[2]] = -np.inf
        x[d, cells[3]] = FILL
        x[d:d + 90, cells[4]] = -0.0
        x[d:d + 3, cells[5]] = np.nan


def _field(T, C, seed, hostile_cells, hostile_days):
    rng = np.random.default_rng(seed)
    x = rng.gamma(0.5, 8.0, size=(T, C)).astype(np.float32)      # continuous: sums are not on a grid
    x[rng.random(x.shape) < 0.35] = 0.0
    x[rng.random(x.shape) < 0.01] = np.nan
    x[:, 0] = np.nan                                             # all NaN
    x[:, 1] = 0.5                                                # constant, on the threshold (_thresholds)
    x[15:40, 2] = np.nan                                         # a NaN run
    x[:, 3] = x[:, 4]                                            # shares the tie thresholds of cell 4
    for cells in hostile_cells:
        _hostile(x, cells, hostile_days)
    return x


def _thresholds(x, w, wstat, n, seed):
    """The constant cell's window statistic (a tie on every window of that cell) and n - 1 window statistics
    that occur in cell 4 (ties in cells 3 and 4)."""
    r = O.window_stat_rule(x[:, [1, 4]], w, wstat)
    vals = r[:, 1][np.isfinite(r[:, 1])]
    rng = np.random.default_rng(seed)
    return [float(r[-1, 0])] + [float(v) for v in rng.choice(vals, n - 1)]


def _layouts(x, names):
    """Device views of the same cells: "aligned" contiguous, "slice" the offset column slice (ldx = C + 1, 4 bytes
    off: one cell per lane), "band" an aligned band view (ldx = C + 4)."""
    import torch
    out = {}
    a = torch.from_numpy(x).cuda()
    for name in names:
        if name == "aligned":
            out[name] = a
        else:
            off = 1 if name == "slice" else 0
            buf = torch.full((x.shape[0], x.shape[1] + (1 if name == "slice" else 4)), 7e9, dtype=torch.float32,
                             device=a.device)
            buf[:, off:off + x.shape[1]] = a
            out[name] = buf[:, off:off + x.shape[1]]
    return out


def _layout_args(v):
    """(C, ldx, 16-byte aligned base) of a device view"""
    return v.shape[1], v.stride(0), v.data_ptr() % 16 == 0


def _spell_kernel(layout, w, ws, r, before):
    C, ldx, al = layout
    return H.spell_instance(C, ldx, w, ST[ws], RL[r], before, aligned_x=al)


def _rolling_kernel(layout, w, ws, s, center):
    C, ldx, al = layout
    return H.rolling_instance(C, ldx, w, ST[ws], ST[s], center, aligned_x=al)


# ------------------------------------------------------------------------------------------------- launches
_FAMILY = ("spell_sumw", "rolling_sumw", "spell_runstat4", "rolling_period_reduce4", "rolling_period_reduce_sel",
           "rolling_period_reduce", "spell_runstat", "spell_mask", "rolling_mean")


def _instance(name):
    """"spell_sumw<5, -1, true>", "rolling_period_reduce4", ... from a demangled or mangled kernel name"""
    import re
    for base in _FAMILY:
        m = re.search(rf"(?<![A-Za-z0-9_]){base}_kernel(?:<([^>]*)>|I((?:L[bi]n?\d+E)+)E)?", name)
        if not m:
            m = re.search(rf"\d{base}_kernel(?:<([^>]*)>|I((?:L[bi]n?\d+E)+)E)?", name)
        if m:
            dem, man = m.groups()
            if man:
                conv = {"b1": "true", "b0": "false"}
                dem = ", ".join(conv.get(a, a[1:].replace("n", "-")) for a in re.findall(r"L([bi]n?\d+)E", man))
            return f"{base}<{dem}>" if dem else base
    return None


class Launches:
    """Records the rolling-family kernels launched inside ``with``; ``seen`` is None when the profiler saw none."""

    def __enter__(self):
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        self._p = profile(activities=[ProfilerActivity.CUDA])
        self._p.__enter__()
        return self

    def __exit__(self, *a):
        import torch
        torch.cuda.synchronize()
        self._p.__exit__(*a)
        names = [e.name for e in self._p.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        kernels = [n for n in names if "kernel" in n.lower() or n.startswith("_Z")]
        self.seen = {i for i in map(_instance, kernels) if i} if kernels else None
        return False


def _witness(rec, expect):
    """Every launch recorded is an expected instance, and every expected instance is recorded.  Late in a long
    pytest process torch.profiler has been seen to lose some CUDA kernel records of a session (never when this
    file runs alone): a missing record is reported as a warning, an unexpected kernel always fails."""
    import warnings
    if rec.seen is None:
        warnings.warn("torch.profiler recorded no kernels: the launched instances are not witnessed")
        return
    assert rec.seen <= expect, sorted(rec.seen - expect)
    if rec.seen != expect:
        warnings.warn(f"torch.profiler recorded no launch of {sorted(expect - rec.seen)}")


# ------------------------------------------------------------------------------------------------- checks
def _check_runs(got, exp, red, msg):
    if red in ("mean", "std"):
        np.testing.assert_allclose(got, exp, rtol=1e-5, atol=0, err_msg=msg)
    else:
        np.testing.assert_array_equal(got, exp, err_msg=msg)


def _check_stat(got, exp, stat, msg):
    if stat in ("sum", "min", "max", "count"):
        np.testing.assert_array_equal(got, exp, err_msg=msg)
    else:
        np.testing.assert_allclose(got, exp, rtol=1e-5, atol=1e-4 if stat in ("std", "var") else 0, equal_nan=True,
                                   err_msg=msg)


def _same_bits(outs, msg):
    for o in outs[1:]:
        np.testing.assert_array_equal(o.view(np.uint32), outs[0].view(np.uint32), err_msg=msg)


def _run_spells(x, views, poff, w, specs, befores, sel=None, msg=""):
    """specs: (wstat, op, thr, reducers).  Runs every (spec, reducer, before) on every view, compares the first
    view with the rule on the cells ``sel`` and all views with each other."""
    from xclim_b200 import device
    xs = x if sel is None else x[:, sel]
    expect = {_spell_kernel(_layout_args(v), w, ws, r, b) for v in views.values()
              for ws, _, _, reds in specs for r in reds for b in befores}
    got = {}
    with Launches() as rec:
        for ws, op, thr, reds in specs:
            for r in reds:
                for b in befores:
                    got[ws, op, thr, r, b] = [device.spell_runstat(v, poff, w, ST[ws], OPC[op], thr, RL[r], b)
                                              for v in views.values()]
    _witness(rec, expect)
    for ws, op, thr, reds in specs:
        mask = O.spell_mask_rule(xs, w, ws, op, thr).astype(np.float32)
        for r in reds:
            for b in befores:
                m = f"{msg} w={w} {ws} {op} {thr!r} {r} before={b}"
                outs = [o.cpu().numpy() for o in got[ws, op, thr, r, b]]
                _same_bits(outs, m)
                exp = O.resample_and_rl(mask, b, O.rle_statistics, poff=poff, reducer=r, window=1).astype(np.float32)
                _check_runs(outs[0] if sel is None else outs[0][:, sel], exp, r, m)
    return expect


def _run_rolling(x, views, poff, w, specs, sel=None, msg=""):
    """specs: (wstat, center, stats)."""
    from xclim_b200 import device
    xs = x if sel is None else x[:, sel]
    expect = {_rolling_kernel(_layout_args(v), w, ws, s, c) for v in views.values()
              for ws, c, stats in specs for s in stats}
    got = {}
    with Launches() as rec:
        for ws, c, stats in specs:
            for s in stats:
                got[ws, c, s] = [device.rolling_period_reduce(v, poff, w, ST[ws], c, ST[s]) for v in views.values()]
    _witness(rec, expect)
    for ws, c, stats in specs:
        vals = O.rolling_rule(xs, w, ws, c)
        for s in stats:
            m = f"{msg} w={w} {ws} center={c} {s}"
            outs = [o.cpu().numpy() for o in got[ws, c, s]]
            for o in outs[1:]:
                np.testing.assert_array_equal(o, outs[0], err_msg=m)
            _check_stat(outs[0] if sel is None else outs[0][:, sel], O.period_stat_rule(vals, poff, s), s, m)
    return expect


# ------------------------------------------------------------------------------------------------- cases
# 425 steps x 24 cells, the hostile cells at 8..13 (the first lanes of their 4-cell groups differ) early in
# the periods starting at 31, 181 and 365
SMALL = dict(T=425, C=24, poff=P_SMALL, hostile=[(8, 9, 10, 11, 12, 13), (18, 19, 21, 22, 15, 23)],
             days=[33, 183, 366])
SMALL_LAYOUTS = ("aligned", "slice", "band")


def _small_field(seed):
    return _field(SMALL["T"], SMALL["C"], seed, SMALL["hostile"], SMALL["days"])


def _spell_specs(w, x, seed):
    """Every operator on sum windows, two on the others, all six reducers; the threshold cycles through the
    tie values."""
    specs = []
    for k, ws in enumerate(WSTATS):
        ops = OPS if ws == "sum" else [OPS[(w + 2 * k) % 6], OPS[(w + 2 * k + 3) % 6]]
        thrs = _thresholds(x, w, ws, len(ops), seed + k)
        specs += [(ws, op, thr, REDUCERS) for op, thr in zip(ops, thrs)]
    return specs


def _small_spell_instances(w):
    views = [(24, 24, True), (24, 25, False), (24, 28, True)]
    return {_spell_kernel(v, w, ws, r, b) for v in views for ws in WSTATS for r in REDUCERS
            for b in (True, False)}


def _small_rolling_specs(w):
    return [(ws, c, STATS) for ws in WSTATS for c in ((False, True) if w % 2 else (False,))]


def _small_rolling_instances(w):
    views = [(24, 24, True), (24, 25, False), (24, 28, True)]
    return {_rolling_kernel(v, w, ws, s, c) for v in views for ws, c, stats in _small_rolling_specs(w)
            for s in stats}


@pytest.mark.parametrize("w", WINDOWS)
def test_spell_small(cuda, w):
    x = _small_field(100 + w)
    views = _layouts(x, SMALL_LAYOUTS)
    got = _run_spells(x, views, P_SMALL, w, _spell_specs(w, x, w), (True, False), msg="small")
    assert got == _small_spell_instances(w)


@pytest.mark.parametrize("w", WINDOWS)
def test_rolling_small(cuda, w):
    x = _small_field(200 + w)
    views = _layouts(x, SMALL_LAYOUTS)
    got = _run_rolling(x, views, P_SMALL, w, _small_rolling_specs(w), msg="small")
    assert got == _small_rolling_instances(w)


def test_rolling_window_is_series(cuda):
    """w = T: one window, longer than every period (the lane kernel: w > 80)."""
    x = _field(90, 24, 7, [(8, 9, 10, 11, 12, 13)], [2])
    views = _layouts(x, SMALL_LAYOUTS)
    poff = np.array([0, 30, 31, 90], np.int32)
    _run_rolling(x, views, poff, 90, [("sum", False, STATS), ("max", False, ["max", "count"])], msg="w=T")
    _run_spells(x, views, poff, 90, [("sum", "<", 1e9, ["max", "count"])], (True, False), msg="w=T")


@pytest.mark.parametrize("w", [1, 3, 7, 12, 80])
def test_three_cells(cuda, w):
    """C = 3: the lane kernels; the hostile cells in every column."""
    x = _field(425, 8, 300 + w, [], [])[:, 4:7].copy()
    for c in range(3):
        d = 33 + 30 * c
        x[d, c] = [np.inf, FILL, -np.inf][c]
    views = _layouts(x, ("aligned", "slice"))
    _run_spells(x, views, P_SMALL, w, [("sum", "<", 0.5 * w, REDUCERS), ("mean", ">=", 2.0, ["max", "count"])],
                (True, False), msg="C=3")
    _run_rolling(x, views, P_SMALL, w, [("sum", False, STATS), ("mean", bool(w % 2), ["max", "min", "mean"])],
                 msg="C=3")


# several CTAs with a partial last one; hostile cells in the first 4-cell groups and in the last CTA
def _wide_cells(C):
    hostile = [(8, 9, 10, 11, 12, 13), (C - 6, C - 5, C - 4, C - 3, C - 2, C - 1)]
    rng = np.random.default_rng(C)
    sel = np.unique(np.concatenate([np.arange(24), [127, 128, 129, 511, 512, 513], rng.choice(C, 24, replace=False),
                                    np.arange(C - 12, C)]))
    return hostile, sel


WIDE = [
    # C, T, poff, layouts, windows
    pytest.param(1028, 730, P_MS, ("aligned", "slice"), (2, 6, 7, 9, 31), id="C1028-MS"),
    pytest.param(1028, 730, P_QS, ("aligned", "band"), (5, 8, 12, 80, 81), id="C1028-QSDEC"),
    pytest.param(2052, 10950, P_YS, ("aligned", "slice", "band"), (3, 10, 80, 81), id="C2052-YS30"),
]


@pytest.mark.parametrize("C,T,poff,layouts,windows", WIDE)
def test_wide(cuda, C, T, poff, layouts, windows):
    import torch
    hostile, sel = _wide_cells(C)
    days = [int(poff[1]) + 2, int(poff[len(poff) // 2]) + 1]
    x = _field(T, C, C + T, hostile, days)
    views = _layouts(x, layouts)
    xs = x[:, sel]
    for w in windows:
        t_sum, t_mean = _thresholds(xs, w, "sum", 2, w), _thresholds(xs, w, "mean", 2, w)
        specs = [("sum", "<", t_sum[0], ["count", "max"]), ("sum", ">=", t_sum[1], ["sum", "mean"]),
                 ("mean", "==", t_mean[0], ["count"]), ("max", ">", 30.0, ["max"])]
        _run_spells(x, views, poff, w, specs, (True, False), sel=sel, msg=f"C={C}")
        rspecs = [("sum", False, ["max", "sum", "count", "mean"]), ("mean", bool(w % 2), ["min", "std"]),
                  ("min", False, ["max"])]
        _run_rolling(x, views, poff, w, rspecs, sel=sel, msg=f"C={C}")
    del views
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------- spell mask
@pytest.mark.parametrize("w", [6, 7, 12])      # either side of BlockStream's sliding switch (w > 6)
def test_spell_mask_season(cuda, w):
    from xclim_b200 import device
    x = _field(730, 24, 400 + w, [(8, 9, 10, 11, 12, 13)], [100, 460])
    doy = np.arange(730) % 365
    keep = ((doy >= 90) & (doy < 250)).astype(np.uint8)
    views = _layouts(x, ("aligned", "slice"))
    for ws in WSTATS:
        for op, thr in zip(("<", ">=", "!="), _thresholds(x, w, ws, 3, w)):
            with Launches() as rec:
                outs = [device.spell_mask(v, w, ST[ws], OPC[op], thr, keep, drop_nan_adjacent=False).cpu().numpy()
                        for v in views.values()]
            _witness(rec, {"spell_mask"})
            exp = np.where(keep[:, None] != 0, O.spell_mask_rule(x, w, ws, op, thr), np.nan).astype(np.float32)
            m = f"w={w} {ws} {op} {thr!r}"
            _same_bits(outs, m)
            np.testing.assert_array_equal(outs[0], exp, err_msg=m)


# ------------------------------------------------------------------------------------------------- controls
@pytest.mark.parametrize("w", [3, 10, 31])
def test_direct_sum_controls(cuda, w):
    """rolling_period_reduce_sel and rolling_mean sum every window directly (window_stat)."""
    from xclim_b200 import device
    x = _small_field(500 + w)
    rng = np.random.default_rng(w)
    keep = (((np.arange(425) % 365) >= 20) & ((np.arange(425) % 365) < 250)) | (rng.random(425) < 0.1)
    views = _layouts(x, ("aligned", "slice"))
    for ws in WSTATS:
        c = bool(w % 2)
        vals = np.where(keep[:, None], O.rolling_rule(x, w, ws, c), np.nan)
        for s in STATS:
            with Launches() as rec:
                outs = [device.rolling_period_reduce_sel(v, P_SMALL, w, ST[ws], c, ST[s], keep.astype(np.uint8))
                        .cpu().numpy() for v in views.values()]
            _witness(rec, {"rolling_period_reduce_sel"})
            for o in outs:
                _check_stat(o, O.period_stat_rule(vals, P_SMALL, s), s, f"sel w={w} {ws} {s}")
    with Launches() as rec:
        outs = [device.rolling_mean(v, w).cpu().numpy() for v in views.values()]
    _witness(rec, {"rolling_mean"})
    exp = O.window_stat_rule(x, w, "mean")
    for o in outs:
        np.testing.assert_array_equal(o, exp, err_msg=f"rolling_mean w={w}")


# ------------------------------------------------------------------------------------------------- coverage
def expected_instances():
    """Every instance the cases above are meant to launch (a CPU check pins it against the dispatch)."""
    out = set()
    for w in WINDOWS:
        out |= _small_spell_instances(w) | _small_rolling_instances(w)
    return out | {"spell_mask"}


def hostile_sliding_instances():
    """The instances that the small cases run with a sliding sum window on hostile data (every case holds hostile
    cells; test_spell_mask_season runs spell_mask at w = 7 and 12)."""
    out = {"spell_mask"}
    for w in WINDOWS:
        out |= {k for k in _small_spell_instances(w) | _small_rolling_instances(w) if H.instance_slides(k, w, ST["sum"])}
    return out
