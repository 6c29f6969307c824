"""CPU oracle for the rain season (indices/_agro.py:790-980 `rain_season`).  TEST INFRASTRUCTURE ONLY.

A literal numpy restatement of the reference's array passes, period by period (``resample(time=freq).map``,
:976), over ``(time, cells)`` arrays: the rolling sums, ``_cumsum_reset(index="first")``, ``runs_with_holes``,
``rle(index="first")``, ``select_time`` (through ``TimeAxis.select_mask``), ``nanargmax`` / ``nanargmin``, the
forward-filled ``start + 1`` mask and ``lazy_indexing``.  It is deliberately not the one-pass scan of
xclim_b200/csrc/rain_season_core.cuh, so that the two check each other.  ``file:line`` is relative to
``/root/reference/src/xclim``.

Two documented choices (DESIGN.md section 4): a window sum is the float64 sum of its values in time order, NaN if
any is NaN, rounded once to float32 (xarray sums in float32); and a start on a period's last step, where the
reference's ``mask[{"time": start + 1}]`` indexes past the period, leaves no step after the start to search.
"""
from __future__ import annotations

import numpy as np


def rolling_sum(a, w):
    """``a.rolling(time=w).sum()`` (min_periods = w, labelled at the window's last step) with the sum rule above."""
    a = np.asarray(a, dtype=np.float32)
    n = a.shape[0]
    out = np.full(a.shape, np.nan, np.float32)
    m = n - w + 1
    if m <= 0:
        return out
    s = np.zeros((m,) + a.shape[1:], np.float64)
    for k in range(w):                                   # time order inside every window
        s = s + a[k:k + m].astype(np.float64)
    out[w - 1:] = s.astype(np.float32)
    return out


def _cumsum_reset(da, index):
    """indices/run_length.py:144-151 (`_cumsum_reset_np`): 100110111 -> 100120123 ("last") or 300210321 ("first")."""
    arr = np.array(da, dtype=np.int64)
    n = arr.shape[0]
    it = range(1, n) if index == "last" else range(n - 2, -1, -1)
    for i in it:
        arr[i] *= arr[i - it.step] + 1
    return arr


def _ffill(a):
    """``DataArray.ffill("time")`` of a float array."""
    a = a.copy()
    for i in range(1, a.shape[0]):
        a[i] = np.where(np.isnan(a[i]), a[i - 1], a[i])
    return a


def runs_with_holes(da_start, window_start, da_stop, window_stop):
    """indices/run_length.py:844-888."""
    start_runs = _cumsum_reset(np.nan_to_num(da_start.astype(np.float64)).astype(np.int64), "first")
    stop_runs = _cumsum_reset(np.nan_to_num(da_stop.astype(np.float64)).astype(np.int64), "first")
    start_positions = np.where(start_runs >= window_start, 1.0, np.nan)
    stop_positions = np.where(stop_runs >= window_stop, 0.0, np.nan)
    runs = np.where(np.isnan(stop_positions), start_positions, stop_positions)    # combine_first
    return np.nan_to_num(_ffill(runs), nan=0.0)


def rle(da):
    """indices/run_length.py:223-272 with index="first": the run length on the first step of every run of values
    > 0, 0 where the value is <= 0, NaN on the other steps of a run."""
    da = np.asarray(da, dtype=np.float64)[::-1]
    cs_s = _cumsum_reset(da, "last").astype(np.float64)
    nxt = np.zeros_like(da)
    nxt[:-1] = da[1:]                                    # da.shift(-1, fill_value=0)
    cs_s = np.where(nxt == 0, cs_s, np.nan)
    out = np.where(da > 0, cs_s, 0.0)
    return out[::-1]


def _get_first_run(run_positions, sel):
    """_agro.py:898-901: the first True of ``run_positions`` among the steps ``sel`` that
    ``select_time(date_bounds=...)`` keeps, NaN when argmax == argmin."""
    arr = np.where(sel[:, None], np.asarray(run_positions, dtype=np.float64), np.nan)
    first = np.nanargmax(arr, axis=0)                    # ValueError when the bounds select nothing
    return np.where(first != np.nanargmin(arr, axis=0), first, np.nan)


def period(pram, pre, sel_start, sel_end, p):
    """Step indices ``(start, end)`` and ``length`` of one period, (C,) float64 each.  ``pram``: (n, C) float32
    amounts; ``pre``, ``sel_start``, ``sel_end``: (n,) bool, the steps that ``select_time`` keeps for the onset
    prefilter (date_min_start .. the period's last day), for ``_get_first_run`` of the start and of the end."""
    n = pram.shape[0]
    with np.errstate(invalid="ignore"):
        # _get_first_run_start, :904-927
        xs = np.where(pre[:, None], pram, np.float32(np.nan))
        da_start = rolling_sum(xs, p["window_wet_start"]) >= p["thresh_wet_start"]
        if p["method_dry_start"] == "per_day":
            da_stop = xs <= p["thresh_dry_start"]
            window_dry = p["window_dry_start"]
        elif p["method_dry_start"] == "total":
            w = p["window_dry_start"]
            r = rolling_sum(xs, w) <= p["thresh_dry_start"]
            da_stop = np.zeros_like(r)                   # shift(-(w - 1), fill_value=False)
            da_stop[:n - (w - 1)] = r[w - 1:]
            window_dry = 1
        else:
            raise ValueError(f"Unknown method_dry_start: {p['method_dry_start']}.")
        events = runs_with_holes(da_start, 1, da_stop, window_dry)
        run_positions = rle(events) >= (p["window_not_dry_start"] + p["window_wet_start"])
        start = _get_first_run(run_positions, sel_start)

        # :950-957, the day after the start and every later day
        start_ind = np.where(np.isnan(start), -1, start + 1).astype(np.int64)
        mask = np.full(pram.shape, np.nan)
        ok = ~np.isnan(start) & (start_ind < n)
        mask[start_ind[ok], np.nonzero(ok)[0]] = 1.0
        mask = ~np.isnan(_ffill(mask))
        y = np.where(mask, pram, np.float32(np.nan))

        # _get_first_run_end, :931-939
        if p["method_dry_end"] == "per_day":
            run_positions = rle(y <= p["thresh_dry_end"]) >= p["window_dry_end"]
        elif p["method_dry_end"] == "total":
            run_positions = rolling_sum(y, p["window_dry_end"]) <= p["thresh_dry_end"]
        else:
            raise ValueError(f"Unknown method_dry_end: {p['method_dry_end']}.")
        end = _get_first_run(run_positions, sel_end)

    length = np.where(~np.isnan(end), end - start, n - start)
    return start, end, length


DEFAULTS = dict(thresh_wet_start=25.0, window_wet_start=3, window_not_dry_start=30, thresh_dry_start=1.0,
                window_dry_start=7, method_dry_start="per_day", date_min_start="05-01", date_max_start="12-31",
                thresh_dry_end=0.0, window_dry_end=20, method_dry_end="per_day", date_min_end="09-01",
                date_max_end="12-31")


def params32(params):
    """The defaults completed by ``params``, thresholds as the float32 values the comparisons use."""
    p = {**DEFAULTS, **params}
    for k in ("thresh_wet_start", "thresh_dry_start", "thresh_dry_end"):
        p[k] = np.float32(p[k])
    return p


def lazy_indexing(doy, idx):
    """core/utils.py:202-276 on the period's ``time.dt.dayofyear``: NaN stays NaN."""
    out = np.full(idx.shape, np.nan)
    ok = ~np.isnan(idx)
    out[ok] = doy[idx[ok].astype(np.int64)]
    return out


def rain_season(pr, ta, freq="YS-JAN", scale=1.0, **params):
    """``(start, end, length)`` as (P, C) float64, plus the step indices ``(start_idx, end_idx)`` inside each
    period.  ``pr``: (T, C) float32 rates; ``scale`` the rate2amount factor to mm; thresholds in mm (Python
    floats, compared in float32 as NEP 50 does)."""
    p = params32(params)
    pram = np.asarray(pr, dtype=np.float32) * np.float32(scale)       # rate2amount(pr, out_units="mm"), :892
    poff = ta.period_offsets(freq)
    res = {k: [] for k in ("start_idx", "end_idx", "start", "end", "length")}
    for a, b in zip(poff[:-1], poff[1:]):
        tp = ta.isel(slice(int(a), int(b)))
        last_doy = f"{int(tp.month[-1]):02d}-{int(tp.day[-1]):02d}"                 # :905
        s, e, length = period(pram[a:b], tp.select_mask(date_bounds=(p["date_min_start"], last_doy)),
                              tp.select_mask(date_bounds=(p["date_min_start"], p["date_max_start"])),
                              tp.select_mask(date_bounds=(p["date_min_end"], p["date_max_end"])), p)
        res["start_idx"].append(s)
        res["end_idx"].append(e)
        res["start"].append(lazy_indexing(tp.doy, s))
        res["end"].append(lazy_indexing(tp.doy, e))
        res["length"].append(length)
    return {k: np.stack(v).astype(np.float64) for k, v in res.items()}
